// kge_topk.cu -- running top-K lists over score tiles (link prediction: ScoreInfer.topK, models/infer.py of the reference,
// without its [H * R * T] score vector and host argsort).
//
// Element (q, j) of a tile S [Q, ld] has score S[q, j] and key qoff[q] + (cbase + j) * cstride; row q feeds list
// g = qgroup[q] (the rows of one list are consecutive within a call).  A list holds the K best elements it has seen, in
// the strict total order (score descending, key ascending); a NaN never enters.  Keys are distinct, so the set is unique
// and the result does not depend on launch geometry or on the order of any atomic.
//
//   k_topk_select  one CTA per (row, 4 096-column segment).  It reads its list's K-th entry once as a threshold, reads
//                  each score once, and keeps the elements that beat the threshold (compacted in shared memory as a
//                  64-bit image: order-preserving uint32 of the score << 12 | (4095 - column), so that within a row a
//                  larger image is a better element: the key grows with the column).  More than K survivors (every
//                  element of a list's first tiles, an all-equal tile): a radix select over the images finds the
//                  exact K-th and only the K best leave.  The CTA's K-th score also raises a per-list bound (atomicMax
//                  of the score image): the list's final K-th cannot be worse, so no CTA of the list needs to hand over
//                  an element below it.  The bound only prunes; which CTA raised it first changes nothing in the result.
//   k_topk_merge   one CTA per list touched by the tile (the CTA of the run's first row): the list and the survivors
//                  of the run's CTAs in a 2 048-entry shared buffer; whenever it could overflow, a bitonic sort keeps the
//                  K best, and the new K-th becomes the filter for the survivors still to come.
#include "kge_common.cuh"

namespace kge {

constexpr int kSelBlock = 256;
constexpr int kSelPer = kTopkSeg / kSelBlock;        // scores per thread
constexpr int kMergeBlock = 512;
constexpr int kMergeCap = 2 * KGE_TOPK_MAX;          // list + one round of survivors, a power of two
static_assert((kMergeCap & (kMergeCap - 1)) == 0 && kMergeCap - KGE_TOPK_MAX >= kMergeBlock, "merge buffer");
static_assert(kTopkSeg == 4096, "the image keeps 12 bits of column");

// order-preserving image of a non-NaN float; -0.0 maps to +0.0's image (the two compare equal)
__device__ __forceinline__ unsigned score_ord(float s) {
  unsigned u = __float_as_uint(s);
  if (s == 0.f) u = 0u;
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// (s, k) comes before (ts, tk) in the list order; tk < 0 is an empty slot, after every element
__device__ __forceinline__ bool topk_before(float s, long long k, float ts, long long tk) {
  return k >= 0 && (tk < 0 || s > ts || (s == ts && k < tk));
}

__global__ void __launch_bounds__(kSelBlock) k_topk_select(TopkParams p) {
  __shared__ unsigned long long s_v[kTopkSeg];
  __shared__ unsigned s_hist[256];
  __shared__ int s_n, s_out, s_k;
  __shared__ unsigned s_digit, s_bound;
  const long long nseg = (p.N + kTopkSeg - 1) / kTopkSeg;
  const long long slot = blockIdx.x;
  const long long q = slot / nseg;
  const long long j0 = (slot % nseg) * kTopkSeg;
  const int n = (int)min((long long)kTopkSeg, p.N - j0);
  const long long g = p.qgroup[q];
  const float ts = p.top_score[g * p.K + p.K - 1];
  const long long tk = p.top_key[g * p.K + p.K - 1];
  const long long key0 = p.qoff[q] + (p.cbase + j0) * p.cstride;
  const float* __restrict__ row = p.S + q * p.ld + j0;
  if (threadIdx.x == 0) s_n = s_out = 0;
  float v[kSelPer];
#pragma unroll
  for (int i = 0; i < kSelPer; ++i) {
    const int j = threadIdx.x + i * kSelBlock;
    v[i] = j < n ? row[j] : __int_as_float(0x7fffffff);
  }
  __syncthreads();
#pragma unroll
  for (int i = 0; i < kSelPer; ++i) {
    const int j = threadIdx.x + i * kSelBlock;
    const float s = v[i];
    if (s == s && (tk < 0 || s > ts || (s == ts && key0 + j * p.cstride < tk)))
      s_v[atomicAdd(&s_n, 1)] = ((unsigned long long)score_ord(s) << 12) | (unsigned)(kTopkSeg - 1 - j);
  }
  __syncthreads();
  const int c = s_n;
  unsigned long long vmin = 0;
  if (c > p.K) {
    // radix select of the K-th largest image: 8-bit digits from the top of the 44 used bits
    unsigned long long prefix = 0;
    int k = p.K;
    for (int shift = 40; shift >= 0; shift -= 8) {
      for (int b = threadIdx.x; b < 256; b += kSelBlock) s_hist[b] = 0;
      __syncthreads();
      for (int i = threadIdx.x; i < c; i += kSelBlock) {
        const unsigned long long x = s_v[i];
        if ((x >> (shift + 8)) == prefix) atomicAdd(&s_hist[(x >> shift) & 255], 1u);
      }
      __syncthreads();
      if (threadIdx.x < 32) {
        const int lane = threadIdx.x;
        unsigned cnt[8], sum = 0;
#pragma unroll
        for (int t = 0; t < 8; ++t) sum += cnt[t] = s_hist[255 - 8 * lane - t];
        unsigned incl = sum;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const unsigned y = __shfl_up_sync(0xffffffffu, incl, o);
          if (lane >= o) incl += y;
        }
        unsigned run = incl - sum;
        if (run < (unsigned)k && (unsigned)k <= incl) {
#pragma unroll
          for (int t = 0; t < 8; ++t) {
            if (run < (unsigned)k && run + cnt[t] >= (unsigned)k) {
              s_digit = 255 - 8 * lane - t;
              s_k = k - (int)run;
            }
            run += cnt[t];
          }
        }
      }
      __syncthreads();
      prefix = (prefix << 8) | s_digit;
      k = s_k;
    }
    vmin = prefix;                   // the images are distinct: exactly K are >= it
    if (threadIdx.x == 0) {
      const unsigned o = (unsigned)(prefix >> 12);
      s_bound = max(atomicMax(p.bound + g, o), o);
    }
  } else if (threadIdx.x == 0) {
    s_bound = *(volatile unsigned*)(p.bound + g);
  }
  __syncthreads();
  const unsigned bnd = s_bound;
  const long long out = slot * p.K;
  for (int i = threadIdx.x; i < c; i += kSelBlock) {
    const unsigned long long x = s_v[i];
    if (x >= vmin && (unsigned)(x >> 12) >= bnd) {
      const int j = kTopkSeg - 1 - (int)(x & (kTopkSeg - 1));
      const int at = atomicAdd(&s_out, 1);
      p.cs[out + at] = row[j];
      p.ck[out + at] = key0 + j * p.cstride;
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) p.cn[slot] = s_out;
}

// sorts ss/sk[0, fill) into list order (bitonic over the next power of two, padded with empty slots)
__device__ void topk_sort(float* ss, long long* sk, int fill) {
  int n = 1;
  while (n < fill) n <<= 1;
  for (int i = fill + threadIdx.x; i < n; i += kMergeBlock) {
    ss[i] = -INFINITY;
    sk[i] = -1;
  }
  __syncthreads();
  for (int k = 2; k <= n; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = threadIdx.x; i < n; i += kMergeBlock) {
        const int l = i ^ j;
        if (l > i) {
          const float a = ss[i], b = ss[l];
          const long long ka = sk[i], kb = sk[l];
          const bool sw = (i & k) == 0 ? topk_before(b, kb, a, ka) : topk_before(a, ka, b, kb);
          if (sw) {
            ss[i] = b; ss[l] = a;
            sk[i] = kb; sk[l] = ka;
          }
        }
      }
      __syncthreads();
    }
  }
}

__global__ void __launch_bounds__(kMergeBlock) k_topk_merge(TopkParams p) {
  __shared__ float s_s[kMergeCap];
  __shared__ long long s_key[kMergeCap];
  __shared__ unsigned long long s_end, s_next;
  __shared__ int s_fill;
  const long long q0 = blockIdx.x;
  const long long g = p.qgroup[q0];
  if (q0 > 0 && p.qgroup[q0 - 1] == g) return;          // not the first row of its list's run
  if (threadIdx.x == 0) s_end = (unsigned long long)p.Q;
  __syncthreads();
  for (long long b = q0 + 1; b < p.Q; b += kMergeBlock) {
    const long long q = b + threadIdx.x;
    const bool stop = q < p.Q && p.qgroup[q] != g;
    if (stop) atomicMin(&s_end, (unsigned long long)q);
    if (__syncthreads_or(stop)) break;
  }
  const long long nseg = (p.N + kTopkSeg - 1) / kTopkSeg;
  const long long first = q0 * nseg, last = (long long)s_end * nseg;     // the run's select CTAs
  const int K = p.K;
  float* __restrict__ ls = p.top_score + g * K;
  long long* __restrict__ lk = p.top_key + g * K;
  for (int i = threadIdx.x; i < K; i += kMergeBlock) {
    s_s[i] = ls[i];
    s_key[i] = lk[i];
  }
  if (threadIdx.x == 0) {
    s_fill = K;
    s_next = (unsigned long long)(first + kMergeBlock / 32);
  }
  const unsigned bnd = p.bound[g];
  __syncthreads();
  float ts = s_s[K - 1];
  long long tk = s_key[K - 1];
  // each warp walks the survivors of one select CTA at a time, 32 per round
  const int lane = threadIdx.x & 31;
  long long sl = first + (threadIdx.x >> 5);
  int cur = 0, cnt = sl < last ? p.cn[sl] : 0;
  while (true) {
    while (sl < last && cur >= cnt) {
      unsigned long long nx = 0;
      if (lane == 0) nx = atomicAdd(&s_next, 1ull);
      sl = (long long)__shfl_sync(0xffffffffu, nx, 0);
      cur = 0;
      cnt = sl < last ? p.cn[sl] : 0;
    }
    if (!__syncthreads_or(sl < last)) break;
    if (s_fill > kMergeCap - kMergeBlock) {
      topk_sort(s_s, s_key, s_fill);
      ts = s_s[K - 1];
      tk = s_key[K - 1];
      __syncthreads();
      if (threadIdx.x == 0) s_fill = K;
      __syncthreads();
    }
    if (sl < last && cur + lane < cnt) {
      const long long e = sl * K + cur + lane;
      const float s = p.cs[e];
      const long long k = p.ck[e];
      if (score_ord(s) >= bnd && topk_before(s, k, ts, tk)) {
        const int at = atomicAdd(&s_fill, 1);
        s_s[at] = s;
        s_key[at] = k;
      }
    }
    cur += 32;
    __syncthreads();
  }
  topk_sort(s_s, s_key, s_fill);
  for (int i = threadIdx.x; i < K; i += kMergeBlock) {
    ls[i] = s_s[i];
    lk[i] = s_key[i];
  }
}

size_t topk_workspace_bytes(long long Q, long long N, int K, long long G) {
  const size_t slots = (size_t)Q * (size_t)((N + kTopkSeg - 1) / kTopkSeg);
  auto up = [](size_t b) { return (b + 255) & ~(size_t)255; };
  return up(slots * K * sizeof(long long)) + up(slots * K * sizeof(float)) + up(slots * sizeof(int)) +
         up((size_t)G * sizeof(unsigned));
}

void topk_carve(TopkParams& p, void* ws) {
  const size_t slots = (size_t)p.Q * (size_t)((p.N + kTopkSeg - 1) / kTopkSeg);
  auto up = [](size_t b) { return (b + 255) & ~(size_t)255; };
  char* c = static_cast<char*>(ws);
  p.ck = reinterpret_cast<long long*>(c);
  c += up(slots * p.K * sizeof(long long));
  p.cs = reinterpret_cast<float*>(c);
  c += up(slots * p.K * sizeof(float));
  p.cn = reinterpret_cast<int*>(c);
  c += up(slots * sizeof(int));
  p.bound = reinterpret_cast<unsigned*>(c);
}

void launch_topk(const LaunchCtx& c, const TopkParams& p) {
  const long long slots = p.Q * ((p.N + kTopkSeg - 1) / kTopkSeg);
  KGE_LAUNCH(c, k_topk_select, (unsigned)slots, kSelBlock, 0, p);
  KGE_LAUNCH(c, k_topk_merge, (unsigned)p.Q, kMergeBlock, 0, p);
}

}  // namespace kge
