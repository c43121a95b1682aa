// kge_sim.cu -- embedding similarity tiles (the reference's dglke_emb_sim: EmbSimInfer.topK of models/infer.py and the
// *_dist functions of models/pytorch/tensor_models.py:59-100), for kge_topk to rank.
//
// S[i, j] = sim(L[i], R[j]) over a block of left rows and a block of right rows, both fp32 row-major [n, dim].
//
//   dot, cosine, ext_jaccard   k_sim_prep reads each row once: its fp32 norm, and its TF32 hi/lo split in the K-major slab
//                              layout of the wgmma kernels (kge_common.cuh: slab_off), zero-padded to a multiple of 32
//                              columns.  k_sim_gemm then runs a 3xTF32 wgmma GEMM (hi*hi + hi*lo + lo*hi, fp32
//                              accumulation) over 128 x 256 output tiles and applies the function to the accumulator
//                              registers:  dot;  dot / (|x| |y|);  dot / (|x|^2 + |y|^2 - dot) with |x|^2 the square of
//                              the fp32 norm, in the reference's order of operations.
//   l1, l2                     k_sim_diff: fp32 CUDA-core tiles in difference form, sum |x_k - y_k| or sqrt(sum (x_k -
//                              y_k)^2), negated.  The expanded form |x|^2 + |y|^2 - 2 x.y of the TransE_l2 score tiles
//                              has an error proportional to |x|^2 + |y|^2, not to the distance: a row against itself
//                              would score about -sqrt(u) |x| instead of -0.0, and near-duplicates (what a similarity
//                              query looks for) would come out in the wrong order.  Here a zero difference sums to an
//                              exact 0, negated to -0.0 as the reference's -th.norm(x - y) gives.
//   kge_sim_pairs              out[i] = sim(L[i], R[i]): one warp per pair, fp32 FMAs.
#include <cuda.h>
#include "kge_common.cuh"
#include "kge_tc.cuh"

namespace kge {

using namespace tc;

namespace {

// ---------------------------------------------------------------------------------------------------- the GEMM route
constexpr int kSimM = 128, kSimN = 256;            // output tile: two consumer warpgroups x 64 rows, 256 columns
constexpr int kSimStages = 2;
constexpr int kSimThreads = 384;                   // warpgroups 0-1: wgmma + epilogue; warpgroup 2: TMA producer (warp 8)
constexpr uint32_t kSimABytes = kSimM * 128u;      // one 32-column block of 128 left rows (hi or lo)
constexpr uint32_t kSimBBytes = kSimN * 128u;      // the same for 256 right rows
constexpr uint32_t kSimStageBytes = 2u * kSimABytes + 2u * kSimBBytes;
constexpr size_t kSimSmem = (size_t)kSimStages * kSimStageBytes + 1024;

struct SimGemmArgs {
  int sim;                 // kge_sim_t (dot, cosine or ext_jaccard)
  int nL, nR, nblk;        // rows of each side, 32-column blocks of the (padded) row
  const float* nl;         // [nL] fp32 norms (cosine, ext_jaccard)
  const float* nr;         // [nR]
  float* S;                // [nL, nR]
};

// One warp per row: the fp32 norm and the TF32 hi/lo split of the row in slab layout [nblk][n][32], zero-padded.
__global__ void __launch_bounds__(256) k_sim_prep(const float* __restrict__ X, long long n, int dim, int nblk,
                                                  float* __restrict__ hi, float* __restrict__ lo, float* __restrict__ nrm) {
  const long long row = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= n) return;
  const float* x = X + row * dim;
  float ss = 0.f;
  for (int b = 0; b < nblk; ++b) {
    const int k = 32 * b + lane;
    const float v = k < dim ? x[k] : 0.f;
    ss = fmaf(v, v, ss);
    float h, l;
    split_tf32(v, h, l);
    const long long o = slab_off(0, nblk, (int)n, (int)row, k);
    hi[o] = h;
    lo[o] = l;
  }
  ss = warp_sum(ss);
  if (lane == 0) nrm[row] = sqrtf(ss);
}

__device__ __forceinline__ float sim_epilogue(int sim, float dot, float nx, float ny) {
  if (sim == KGE_SIM_COSINE) return dot / (nx * ny);
  if (sim == KGE_SIM_EXT_JACCARD) return dot / ((nx * nx + ny * ny) - dot);
  return dot;
}

// S tile [128 x 256] = sim(L rows, R rows).  Roles are split per warpgroup (warpgroup 2 produces, 0 and 1 consume), so
// the wgmma code sits in a warpgroup-uniform branch; the row is padded to whole 32-column blocks, so every k-block has
// four k-steps and the fence..commit group has no guard inside it.
__global__ void __launch_bounds__(kSimThreads, 1)
k_sim_gemm(const __grid_constant__ CUtensorMap tLh, const __grid_constant__ CUtensorMap tLl,
           const __grid_constant__ CUtensorMap tRh, const __grid_constant__ CUtensorMap tRl, SimGemmArgs g) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t full[kSimStages], empty[kSimStages];
  __shared__ float s_nl[kSimM], s_nr[kSimN];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m0 = blockIdx.x * kSimM, n0 = blockIdx.y * kSimN;
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  const bool norms = g.sim != KGE_SIM_DOT;
  if (threadIdx.x == 0) {
    for (int s = 0; s < kSimStages; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 8); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  for (int t = threadIdx.x; t < kSimM + kSimN; t += kSimThreads) {
    if (t < kSimM) s_nl[t] = (norms && m0 + t < g.nL) ? g.nl[m0 + t] : 1.f;
    else s_nr[t - kSimM] = (norms && n0 + t - kSimM < g.nR) ? g.nr[n0 + t - kSimM] : 1.f;
  }
  __syncthreads();

  if (warp >= 8) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 56;");
    if (warp == 8) {
      for (int kb = 0; kb < g.nblk; ++kb) {
        const int s = kb % kSimStages;
        mbar_wait(&empty[s], ((kb / kSimStages) & 1) ^ 1);
        uint8_t* st = smem + (size_t)s * kSimStageBytes;
        if (elect_one()) {
          mbar_expect_tx(&full[s], kSimStageBytes);
          // slab layout: TMA row of (32-column block kb, row r) = kb * n + r
          tma_load_2d(st, &tLh, &full[s], 0, kb * g.nL + m0);
          tma_load_2d(st + kSimABytes, &tLl, &full[s], 0, kb * g.nL + m0);
          tma_load_2d(st + 2 * kSimABytes, &tRh, &full[s], 0, kb * g.nR + n0);
          tma_load_2d(st + 2 * kSimABytes + kSimBBytes, &tRl, &full[s], 0, kb * g.nR + n0);
        }
        __syncwarp();
      }
    }
  } else {
    asm volatile("setmaxnreg.inc.sync.aligned.u32 224;");
    const int wg = warp >> 2;
    float acc[kSimN / 2];
#pragma unroll
    for (int i = 0; i < kSimN / 2; ++i) acc[i] = 0.f;
    for (int kb = 0; kb < g.nblk; ++kb) {
      const int s = kb % kSimStages;
      mbar_wait(&full[s], (kb / kSimStages) & 1);
      const uint32_t st = smem_u32(smem + (size_t)s * kSimStageBytes);
      const uint64_t dAh = make_desc(st + wg * 8192u), dAl = make_desc(st + kSimABytes + wg * 8192u);
      const uint64_t dBh = make_desc(st + 2 * kSimABytes), dBl = make_desc(st + 2 * kSimABytes + kSimBBytes);
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
        const uint64_t o = (uint64_t)(ks * 2);     // K-major: +32 bytes per k-step inside the 128-byte swizzle span
        wgmma_ss<kSimN>(acc, dAh + o, dBh + o, 1u);
        wgmma_ss<kSimN>(acc, dAh + o, dBl + o, 1u);
        wgmma_ss<kSimN>(acc, dAl + o, dBh + o, 1u);
      }
      wgmma_commit();
      if (kb > 0) {
        wgmma_wait<1>();                           // the previous k-block has retired: its stage is free
        if (lane == 0) mbar_arrive(&empty[(kb - 1) % kSimStages]);
      }
    }
    wgmma_wait<0>();
    reg_fence(acc);
    // accumulator fragment: rows r, r + 8 (r = 16 (warp % 4) + lane / 4 within the warpgroup's 64), columns
    // 8 j + 2 (lane % 4) + {0, 1}
    const int q = lane & 3;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int ml = wg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * h;
      const int m = m0 + ml;
      if (m >= g.nL) continue;
      const float nx = s_nl[ml];
      float* row = g.S + (long long)m * g.nR;
#pragma unroll
      for (int j = 0; j < kSimN / 8; ++j) {
        const int c = 8 * j + 2 * q, n = n0 + c;
        if (n < g.nR) row[n] = sim_epilogue(g.sim, acc[4 * j + 2 * h], nx, s_nr[c]);
        if (n + 1 < g.nR) row[n + 1] = sim_epilogue(g.sim, acc[4 * j + 2 * h + 1], nx, s_nr[c + 1]);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------- the difference route
constexpr int kDT = 64;       // tile edge
constexpr int kDK = 16;       // slab depth
constexpr int kDLD = kDT + 4; // padded leading dimension (keeps float4 alignment)

// S[i, j] = -sum |L_ik - R_jk| (L1) or -sqrt(sum (L_ik - R_jk)^2) (L2).  64 x 64 outputs per CTA, 256 threads, 4 x 4
// register micro-tile, slabs stored transposed ([k][row]) so that the inner loop reads two float4 per 16 pairs.  Rows
// are read with scalar loads: any dim, any row alignment.
template <bool L2>
__global__ void __launch_bounds__(256) k_sim_diff(const float* __restrict__ L, long long nL, const float* __restrict__ R,
                                                  long long nR, int dim, float* __restrict__ S) {
  __shared__ __align__(16) float As[kDK][kDLD];
  __shared__ __align__(16) float Bs[kDK][kDLD];
  const long long i0 = (long long)blockIdx.y * kDT, j0 = (long long)blockIdx.x * kDT;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int lk = threadIdx.x & 15, lr = threadIdx.x >> 4;     // loader: column k0 + lk of rows lr + 16 p
  float acc[4][4];
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int c = 0; c < 4; ++c) acc[r][c] = 0.f;
  // rows lr + 16 p of each side that exist (bit p), read at column k0 + lk through one pointer per side: padding is zero
  // on both sides, so it adds |0 - 0| = 0
  unsigned lok = 0, rok = 0;
#pragma unroll
  for (int p = 0; p < 4; ++p) {
    lok |= (i0 + lr + 16 * p < nL) ? 1u << p : 0u;
    rok |= (j0 + lr + 16 * p < nR) ? 1u << p : 0u;
  }
  const long long step16 = 16LL * dim;
  const float* lp = L + (i0 + lr) * dim + lk;
  const float* rp = R + (j0 + lr) * dim + lk;
  for (int k0 = 0; k0 < dim; k0 += kDK, lp += kDK, rp += kDK) {
    const bool kin = k0 + lk < dim;
#pragma unroll
    for (int p = 0; p < 4; ++p) {
      As[lk][lr + 16 * p] = (kin && (lok >> p & 1u)) ? lp[p * step16] : 0.f;
      Bs[lk][lr + 16 * p] = (kin && (rok >> p & 1u)) ? rp[p * step16] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < kDK; ++kk) {
      const float4 a4 = *reinterpret_cast<const float4*>(&As[kk][ty * 4]);
      const float4 b4 = *reinterpret_cast<const float4*>(&Bs[kk][tx * 4]);
      const float aa[4] = {a4.x, a4.y, a4.z, a4.w}, bb[4] = {b4.x, b4.y, b4.z, b4.w};
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          const float d = aa[r] - bb[c];
          if (L2) acc[r][c] = fmaf(d, d, acc[r][c]);
          else acc[r][c] += fabsf(d);
        }
    }
    __syncthreads();
  }
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const long long i = i0 + ty * 4 + r;
    if (i >= nL) continue;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const long long j = j0 + tx * 4 + c;
      if (j < nR) S[i * nR + j] = -(L2 ? sqrtf(acc[r][c]) : acc[r][c]);
    }
  }
}

// ---------------------------------------------------------------------------------------------------------- pairs
__global__ void __launch_bounds__(256) k_sim_pairs(int sim, const float* __restrict__ L, const float* __restrict__ R,
                                                   long long n, int dim, float* __restrict__ out) {
  const long long i = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (i >= n) return;
  const float* x = L + i * dim;
  const float* y = R + i * dim;
  float a = 0.f, xx = 0.f, yy = 0.f;     // l1: sum |d|, l2: sum d^2, else dot; |x|^2, |y|^2
  for (int k = lane; k < dim; k += 32) {
    const float u = x[k], v = y[k];
    if (sim == KGE_SIM_L1) {
      a += fabsf(u - v);
    } else if (sim == KGE_SIM_L2) {
      const float d = u - v;
      a = fmaf(d, d, a);
    } else {
      a = fmaf(u, v, a);
      xx = fmaf(u, u, xx);
      yy = fmaf(v, v, yy);
    }
  }
  a = warp_sum(a);
  xx = warp_sum(xx);
  yy = warp_sum(yy);
  if (lane != 0) return;
  float s;
  if (sim == KGE_SIM_L1) s = -a;
  else if (sim == KGE_SIM_L2) s = -sqrtf(a);
  else s = sim_epilogue(sim, a, sqrtf(xx), sqrtf(yy));
  out[i] = s;
}

}  // namespace

bool sim_uses_gemm(int sim) { return sim == KGE_SIM_DOT || sim == KGE_SIM_COSINE || sim == KGE_SIM_EXT_JACCARD; }

size_t sim_workspace_bytes(long long nL, long long nR, int dim) {
  const size_t nblk = (size_t)slab_blocks(dim);
  auto up = [](size_t b) { return (b + 1023) & ~(size_t)1023; };
  return 2 * up((size_t)nL * nblk * 32 * sizeof(float)) + 2 * up((size_t)nR * nblk * 32 * sizeof(float)) +
         up((size_t)nL * sizeof(float)) + up((size_t)nR * sizeof(float));
}

int launch_sim_tile(const LaunchCtx& c, int sim, const float* L, long long nL, const float* R, long long nR, int dim,
                    float* S, void* ws) {
  if (!sim_uses_gemm(sim)) {
    const dim3 grid(ceil_div(nR, kDT), ceil_div(nL, kDT));
    if (sim == KGE_SIM_L2) KGE_LAUNCH(c, k_sim_diff<true>, grid, 256, 0, L, nL, R, nR, dim, S);
    else KGE_LAUNCH(c, k_sim_diff<false>, grid, 256, 0, L, nL, R, nR, dim, S);
    return KGE_OK;
  }
  const int nblk = slab_blocks(dim);
  auto up = [](size_t b) { return (b + 1023) & ~(size_t)1023; };
  char* p = static_cast<char*>(ws);
  float* Lh = reinterpret_cast<float*>(p); p += up((size_t)nL * nblk * 32 * sizeof(float));
  float* Ll = reinterpret_cast<float*>(p); p += up((size_t)nL * nblk * 32 * sizeof(float));
  float* Rh = reinterpret_cast<float*>(p); p += up((size_t)nR * nblk * 32 * sizeof(float));
  float* Rl = reinterpret_cast<float*>(p); p += up((size_t)nR * nblk * 32 * sizeof(float));
  float* nl = reinterpret_cast<float*>(p); p += up((size_t)nL * sizeof(float));
  float* nr = reinterpret_cast<float*>(p);
  KGE_LAUNCH(c, k_sim_prep, ceil_div(nL, 8), 256, 0, L, nL, dim, nblk, Lh, Ll, nl);
  KGE_LAUNCH(c, k_sim_prep, ceil_div(nR, 8), 256, 0, R, nR, dim, nblk, Rh, Rl, nr);
  CUtensorMap tLh, tLl, tRh, tRl;
  if (tc_make_map(&tLh, Lh, (long long)nblk * nL, 32, kSimM) || tc_make_map(&tLl, Ll, (long long)nblk * nL, 32, kSimM) ||
      tc_make_map(&tRh, Rh, (long long)nblk * nR, 32, kSimN) || tc_make_map(&tRl, Rl, (long long)nblk * nR, 32, kSimN))
    return KGE_ERR_CUDA;
  if (int rc = smem_optin((const void*)k_sim_gemm, kSimSmem)) return rc;
  SimGemmArgs g{sim, (int)nL, (int)nR, nblk, nl, nr, S};
  const dim3 grid(ceil_div(nL, kSimM), ceil_div(nR, kSimN));
  KGE_LAUNCH(c, k_sim_gemm, grid, kSimThreads, kSimSmem, tLh, tLl, tRh, tRl, g);
  return KGE_OK;
}

void launch_sim_pairs(const LaunchCtx& c, int sim, const float* L, const float* R, long long n, int dim, float* out) {
  KGE_LAUNCH(c, k_sim_pairs, ceil_div(n, 8), 256, 0, sim, L, R, n, dim, out);
}

}  // namespace kge
