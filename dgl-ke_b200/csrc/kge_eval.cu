// kge_eval.cu -- filtered ranking of evaluation queries over score tiles (general_models.py:462-485 of the reference):
//
//   rank_q = 1 + #{ j : S[q, j] >= pos[q]  and  candidate j is not a known triple of query q }
//
// The scores come from kge_score_neg, one tile at a time: a block of rows of one shard (full-entity evaluation, the
// candidates of column j are the ids base + j) or the gathered rows of a chunk's sampled candidates (explicit ids).
// The known triples are a sorted index per corruption side -- keys = kept_entity * n_rel + rel, vals = the corrupted
// side's entity ids, sorted and distinct within a key -- so no [queries, candidates] mask exists anywhere.
//
//   k_rank_count   one CTA per (query, column segment); adds its hits to cnt[q] (integers: the atomics' order is free)
//     range ids      counts the segment's hits, then takes back those of the known ids that fall inside the segment's
//                    id range (two binary searches inside vals[lo, hi) bound them): O(segment + known ids in it)
//     explicit ids   looks every hit column's id up in vals[lo, hi): a duplicate column of a known id is excluded too
//   k_rank_finish  rank = cnt + 1, optionally stored, and {sum 1/r, sum r, #r<=1, #r<=3, #r<=10, #ranks} added to a
//                  double[6] accumulator: per-thread strided sums, a fixed tree, one thread adds -- bitwise reproducible
#include "kge_common.cuh"

namespace kge {

constexpr int kRankBlock = 256;
constexpr int kRankSeg = 1024;        // columns per CTA: a batch of 8 queries on a 64k-column block is 512 CTAs
constexpr int kFinishBlock = 512;

// first index in [lo, hi) whose key is >= k (lower) or > k (upper)
template <class T, bool UPPER>
__device__ __forceinline__ long long bsearch(const T* __restrict__ a, long long lo, long long hi, long long k) {
  while (lo < hi) {
    const long long m = (lo + hi) >> 1;
    const long long v = (long long)a[m];
    if (UPPER ? (v <= k) : (v < k)) lo = m + 1;
    else hi = m;
  }
  return lo;
}

__global__ void __launch_bounds__(kRankBlock) k_rank_count(RankParams p) {
  __shared__ long long s_range[2];
  __shared__ long long s_part[kRankBlock / 32];
  const long long nseg = (p.N + kRankSeg - 1) / kRankSeg;
  const long long q = blockIdx.x / nseg;
  const long long j0 = (blockIdx.x % nseg) * kRankSeg;
  const long long j1 = min(j0 + kRankSeg, p.N);
  const float ps = p.pos[q];
  const float* __restrict__ row = p.S + q * p.ld;
  if (threadIdx.x == 0) {
    long long lo = 0, hi = 0;
    if (p.keys) {
      const long long key = p.kept[q] * p.n_rel + p.rel[q];
      lo = bsearch<long long, false>(p.keys, 0, p.n_keys, key);
      hi = bsearch<long long, true>(p.keys, lo, p.n_keys, key);
      if (!p.cand && lo < hi) {     // range ids: only the known ids inside [base + j0, base + j1)
        const long long a = bsearch<int, false>(p.vals, lo, hi, p.base + j0);
        hi = bsearch<int, false>(p.vals, a, hi, p.base + j1);
        lo = a;
      }
    }
    s_range[0] = lo;
    s_range[1] = hi;
  }
  __syncthreads();
  const long long lo = s_range[0], hi = s_range[1];
  long long c = 0;
  if (!p.cand) {
    for (long long j = j0 + threadIdx.x; j < j1; j += kRankBlock) c += row[j] >= ps;
    for (long long k = lo + threadIdx.x; k < hi; k += kRankBlock) c -= row[(long long)p.vals[k] - p.base] >= ps;
  } else {
    const long long* __restrict__ ids = p.cand + (q / p.chunk) * p.N;
    for (long long j = j0 + threadIdx.x; j < j1; j += kRankBlock) {
      if (!(row[j] >= ps)) continue;
      bool known = false;
      if (lo < hi) {
        const long long id = ids[j];
        const long long k = bsearch<int, false>(p.vals, lo, hi, id);
        known = k < hi && (long long)p.vals[k] == id;
      }
      c += !known;
    }
  }
  for (int o = 16; o; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
  if ((threadIdx.x & 31) == 0) s_part[threadIdx.x >> 5] = c;
  __syncthreads();
  if (threadIdx.x == 0) {
    long long t = 0;
    for (int w = 0; w < kRankBlock / 32; ++w) t += s_part[w];
    if (t) atomicAdd((unsigned long long*)(p.cnt + q), (unsigned long long)t);
  }
}

__global__ void __launch_bounds__(kFinishBlock) k_rank_finish(const long long* __restrict__ cnt, long long Q,
                                                             long long* __restrict__ rank_out, double* __restrict__ acc) {
  __shared__ double s[5][kFinishBlock];
  double v[5] = {0.0, 0.0, 0.0, 0.0, 0.0};
  for (long long q = threadIdx.x; q < Q; q += kFinishBlock) {
    const long long r = cnt[q] + 1;
    if (rank_out) rank_out[q] = r;
    const double rd = (double)r;
    v[0] += 1.0 / rd;
    v[1] += rd;
    v[2] += r <= 1;
    v[3] += r <= 3;
    v[4] += r <= 10;
  }
  for (int i = 0; i < 5; ++i) s[i][threadIdx.x] = v[i];
  __syncthreads();
  for (int w = kFinishBlock / 2; w > 0; w >>= 1) {
    if (threadIdx.x < w)
      for (int i = 0; i < 5; ++i) s[i][threadIdx.x] += s[i][threadIdx.x + w];
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    for (int i = 0; i < 5; ++i) acc[i] += s[i][0];
    acc[5] += (double)Q;
  }
}

void launch_rank_count(const LaunchCtx& c, const RankParams& p) {
  const long long blocks = p.Q * ((p.N + kRankSeg - 1) / kRankSeg);
  KGE_LAUNCH(c, k_rank_count, (unsigned)blocks, kRankBlock, 0, p);
}

void launch_rank_finish(const LaunchCtx& c, const long long* cnt, long long Q, long long* rank_out, double* acc) {
  KGE_LAUNCH(c, k_rank_finish, 1, kFinishBlock, 0, cnt, Q, rank_out, acc);
}

}  // namespace kge
