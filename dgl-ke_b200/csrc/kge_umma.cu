// kge_umma.cu -- stand-alone wgmma (Hopper warpgroup MMA) engine (the file and its umma_* entry points keep their names) for the three chunked contractions of the
// bilinear / L2 models (TransE_l2, DistMult, ComplEx, RESCAL):
//
//   GEMM1  S[c]  = A[c]   . Bn[c]^T     (Cs x Ns, K = D)    operands: A, Bn slabs
//   GEMM2  GA[c] = V[c]   . Bn[c]       (Cs x D,  K = Ns)   operands: V slabs, Bn^T slabs
//   GEMM3  GB[c] = V[c]^T . A[c]        (Ns x D,  K = Cs)   operands: V^T slabs, A^T slabs
//
// wgmma reads TF32 operands from shared memory K-major only, so the producers (k_prep / k_loss) write every operand in
// both orientations (kge_common.cuh: slab_off / slabT_off) and all three GEMMs are the same K-major x K-major kernel.
// fp32 fidelity on TF32 tensor cores: every operand is split x = hi + lo (both rounded to TF32) by its producer
// (kge_common.cuh:split_tf32) and each k-step issues hi*hi + hi*lo + lo*hi (3xTF32), accumulating in fp32 registers.
//
// One CTA per 128 x 128 output tile: warpgroups 0 and 1 each own 64 rows (wgmma m64n128k8, accumulator in registers,
// epilogue straight from the fragments), warp 8 = TMA producer (cp.async.bulk.tensor over the contiguous slab layout,
// 128B swizzle, 3-stage mbarrier pipeline).
#include <cuda.h>
#include <cstdio>
#include <cstdlib>
#include "kge_common.cuh"
#include "kge_tc.cuh"

namespace kge {

using namespace tc;

namespace {

constexpr int kBlockK = 32;                 // fp32 elements per k-block = one 128-byte swizzle span
constexpr int kMmaK = 8;                    // tf32: 32 bytes per MMA k-step
constexpr int kTileM = 128, kTileN = 128;
constexpr int kStages = 3;
constexpr int kThreads = 384;                // warps 0..7 MMA + epilogue (two warpgroups), warp 8 TMA producer
constexpr uint32_t kTileBytes = 128 * 128;   // one operand tile (hi or lo): 128 rows x 128 B
constexpr uint32_t kStageBytes = 4 * kTileBytes;

enum { G_SCORE = 0, G_GA = 1, G_GB = 2 };

struct GemmArgs {
  int mode;              // G_SCORE / G_GA / G_GB
  int C;                 // chunks
  int M, N, K;           // per-chunk extents (rows of A, rows of B, contraction)
  int a_nblk, a_R;       // slab geometry of the A operand matrix: 32-column blocks per chunk, rows per block
  int b_nblk, b_R;       // same for the B operand matrix
  int model;
  float gamma, reg_coef;
  int reg_norm;
  int Cs, Ns, D;
  // epilogue pointers
  float* out;            // SCORE: S [B,Ns] ; GA: GA [B,D] ; GB: Bn [Nn,D] (in place)
  float* out2;           // SCORE: Vdist (TransE_l2)
  const float* a2;       // SCORE l2
  const float* b2;
  const float* colsum;   // GB l2
};

// smem layout per stage: [A_hi | A_lo | B_hi | B_lo], each tile 16 KB, 1024-byte aligned
template <int MODE>
__global__ void __launch_bounds__(kThreads, 1)
k_wgmma_gemm(const __grid_constant__ CUtensorMap tmAh, const __grid_constant__ CUtensorMap tmAl,
             const __grid_constant__ CUtensorMap tmBh, const __grid_constant__ CUtensorMap tmBl, GemmArgs g) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t full_bar[kStages], empty_bar[kStages];
  __shared__ __align__(16) float b2s[kTileN];     // |b_j|^2 of this tile's negatives (score epilogue)

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int c = blockIdx.z;
  const int m0 = blockIdx.y * kTileM;                 // row offset inside the chunk (M dimension)
  const int n0 = blockIdx.x * kTileN;                 // column offset (N dimension)
  const int num_kb = (g.K + kBlockK - 1) / kBlockK;
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);

  if (threadIdx.x == 0) {
    for (int s = 0; s < kStages; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 8); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp == 8) {
    // ===================== TMA producer (all lanes run the loop, one elected lane issues) =====================
    for (int kb = 0; kb < num_kb; ++kb) {
      const int s = kb % kStages;
      const uint32_t ph = (kb / kStages) & 1;
      mbar_wait(&empty_bar[s], ph ^ 1);
      uint8_t* st = smem + (size_t)s * kStageBytes;
      if (elect_one()) {
        mbar_expect_tx(&full_bar[s], kStageBytes);
        // slab layout: row coordinate of (chunk c, 32-column block blk, row r) = (c * nblk + blk) * R + r; x = 0
        const int ya = (c * g.a_nblk + kb) * g.a_R + m0;
        const int yb = (c * g.b_nblk + kb) * g.b_R + n0;
        tma_load_2d(st, &tmAh, &full_bar[s], 0, ya);
        tma_load_2d(st + kTileBytes, &tmAl, &full_bar[s], 0, ya);
        tma_load_2d(st + 2 * kTileBytes, &tmBh, &full_bar[s], 0, yb);
        tma_load_2d(st + 3 * kTileBytes, &tmBl, &full_bar[s], 0, yb);
      }
      __syncwarp();
    }
  } else if (warp < 8) {
    // ===================== MMA + epilogue: warpgroup wg owns rows [64 wg, 64 wg + 64) of the tile =====================
    const int wg = warp >> 2;
    const bool l2 = g.model == KGE_TRANSE_L2;
    if (MODE == G_SCORE && l2) {
      // stage the tile's |b_j|^2 once (every row of the tile needs all of them) while the first loads are in flight
      const int et = threadIdx.x;
      if (et < kTileN) b2s[et] = (n0 + et < g.N) ? g.b2[(long long)c * g.Ns + n0 + et] : 0.f;
      asm volatile("bar.sync 1, 256;" ::: "memory");   // the 8 consumer warps only
    }
    float acc[kTileN / 2];
#pragma unroll
    for (int i = 0; i < kTileN / 2; ++i) acc[i] = 0.f;
    for (int kb = 0; kb < num_kb; ++kb) {
      const int s = kb % kStages;
      mbar_wait(&full_bar[s], (kb / kStages) & 1);
      const uint32_t st = smem_u32(smem + (size_t)s * kStageBytes);
      const uint64_t dAh = make_desc(st + wg * 8192u), dAl = make_desc(st + kTileBytes + wg * 8192u);
      const uint64_t dBh = make_desc(st + 2 * kTileBytes), dBl = make_desc(st + 3 * kTileBytes);
      const int kleft = g.K - kb * kBlockK;
      const int ksteps = kleft >= kBlockK ? kBlockK / kMmaK : kleft / kMmaK;   // K % 8 == 0 guaranteed
      wgmma_fence();
      for (int ks = 0; ks < ksteps; ++ks) {
        const uint64_t o = (uint64_t)(ks * 2);     // +32 bytes per k-step inside the 128-byte swizzle span
        wgmma_ss<kTileN>(acc, dAh + o, dBh + o, 1u);
        wgmma_ss<kTileN>(acc, dAh + o, dBl + o, 1u);
        wgmma_ss<kTileN>(acc, dAl + o, dBh + o, 1u);
      }
      wgmma_commit();
      if (kb > 0) {
        wgmma_wait<1>();                             // the previous k-block's MMAs have retired: its stage is free
        if (lane == 0) mbar_arrive(&empty_bar[(kb - 1) % kStages]);
      }
    }
    wgmma_wait<0>();
    reg_fence(acc);

    // epilogue from the accumulator fragment: rows r0, r0 + 8; columns 8 j + 2 (lane % 4) + {0, 1}
    const int q = lane & 3;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int m = m0 + wg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * h;
      if (m >= g.M) continue;
      if (MODE == G_SCORE) {
        const long long gi = (long long)c * g.Cs + m;
        const float a2v = l2 ? g.a2[gi] : 0.f;
#pragma unroll
        for (int j = 0; j < kTileN / 8; ++j) {
          const int col = 8 * j + 2 * q, n = n0 + col;
          if (n >= g.N) continue;
          float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
          if (l2) {
            // batched_l2_dist (score_fun.py:26-34): (|b|^2 - 2 a.b) + |a|^2, clamp, sqrt
            const float d0 = sqrtf(fmaxf(fmaf(-2.f, v0, b2s[col]) + a2v, 1e-30f));
            const float d1 = sqrtf(fmaxf(fmaf(-2.f, v1, b2s[col + 1]) + a2v, 1e-30f));
            *reinterpret_cast<float2*>(g.out2 + gi * g.Ns + n) = make_float2(d0, d1);
            v0 = g.gamma - d0; v1 = g.gamma - d1;
          }
          *reinterpret_cast<float2*>(g.out + gi * g.Ns + n) = make_float2(v0, v1);
        }
      } else if (MODE == G_GA) {
        float* row = g.out + ((long long)c * g.Cs + m) * g.D;
#pragma unroll
        for (int j = 0; j < kTileN / 8; ++j) {
          const int k = n0 + 8 * j + 2 * q;
          if (k < g.N) *reinterpret_cast<float2*>(row + k) = make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
        }
      } else {  // G_GB: gradient of the negative rows, written over the gathered rows
        float* row = g.out + ((long long)c * g.Ns + m) * g.D;
        const float cs = l2 ? g.colsum[(long long)c * g.Ns + m] : 0.f;
#pragma unroll
        for (int j = 0; j < kTileN / 8; ++j) {
          const int k = n0 + 8 * j + 2 * q;
          if (k >= g.N) continue;
          const float2 b = *reinterpret_cast<const float2*>(row + k);
          float g0 = acc[4 * j + 2 * h], g1 = acc[4 * j + 2 * h + 1];
          if (l2) { g0 = fmaf(-cs, b.x, g0); g1 = fmaf(-cs, b.y, g1); }     // sum_i V_ij a_i - (sum_i V_ij) b_j
          *reinterpret_cast<float2*>(row + k) = make_float2(g0 + reg_grad(b.x, g.reg_norm, g.reg_coef),
                                                            g1 + reg_grad(b.y, g.reg_norm, g.reg_coef));
        }
      }
    }
  }
}

// ---- host side ----------------------------------------------------------------------------------
typedef CUresult (*encode_fn_t)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

encode_fn_t get_encode() {
  static encode_fn_t fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = (encode_fn_t)p;
  }
  return fn;
}

// cuTensorMapEncodeTiled is a host-side driver call per map; the workspace matrices keep their
// addresses between steps, so the encoded maps are cached (per host thread).
struct MapKey { const void* base; long long rows, cols; int box_rows; int dev; };
struct MapCache {
  static constexpr int kN = 64;
  MapKey keys[kN];
  CUtensorMap maps[kN];
  int n = 0, next = 0;
};
thread_local MapCache g_maps;

template <int MODE>
int launch_gemm(const LaunchCtx& c, const CUtensorMap& ah, const CUtensorMap& al, const CUtensorMap& bh,
                const CUtensorMap& bl, const GemmArgs& g) {
  const size_t smem = (size_t)kStages * kStageBytes + 1024;
  if (int rc = smem_optin((const void*)k_wgmma_gemm<MODE>, smem)) return rc;
  dim3 grid((g.N + kTileN - 1) / kTileN, (g.M + kTileM - 1) / kTileM, g.C);
  const char* nm = MODE == G_SCORE ? "k_wgmma_gemm<score S=A.Bn^T>"
                                   : (MODE == G_GA ? "k_wgmma_gemm<grad_a GA=V.Bn>" : "k_wgmma_gemm<grad_b GB=V^T.A>");
  KGE_LAUNCH_NAMED(c, nm, (k_wgmma_gemm<MODE>), grid, kThreads, smem, ah, al, bh, bl, g);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(KGE_ERR_CUDA, "wgmma gemm launch: %s", cudaGetErrorString(e));
  return KGE_OK;
}

}  // namespace

int tc_make_map(CUtensorMap* m, const float* base, long long rows, long long cols, int box_rows) {
  MapCache& mc = g_maps;
  int dev = 0;
  cudaGetDevice(&dev);
  for (int i = 0; i < mc.n; ++i) {
    const MapKey& k = mc.keys[i];
    if (k.base == base && k.rows == rows && k.cols == cols && k.box_rows == box_rows && k.dev == dev) {
      *m = mc.maps[i];
      return KGE_OK;
    }
  }
  encode_fn_t enc = get_encode();
  if (!enc) return fail(KGE_ERR_CUDA, "cuTensorMapEncodeTiled not available");
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)cols * 4};
  cuuint32_t box[2] = {32u, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1u, 1u};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, (void*)base, dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS)
    return fail(KGE_ERR_CUDA, "cuTensorMapEncodeTiled failed (%d) rows=%lld cols=%lld box_rows=%d", (int)r, rows, cols, box_rows);
  int slot = mc.n < MapCache::kN ? mc.n++ : (mc.next++ % MapCache::kN);
  mc.keys[slot] = MapKey{base, rows, cols, box_rows, dev};
  mc.maps[slot] = *m;
  return KGE_OK;
}

bool umma_supported(const StepParams& p) {
  const bool model_ok = p.model == KGE_TRANSE_L2 || p.model == KGE_DISTMULT || p.model == KGE_COMPLEX || p.model == KGE_RESCAL;
  return model_ok && (p.D % 8 == 0) && (p.Cs % 8 == 0) && (p.Ns % 8 == 0) && p.D >= 32 && p.Cs >= 8 && p.Ns >= 8 &&
         prep_stage_fits(p.D);     // k_prep writes the transposed slabs from 32 rows staged in shared memory
}

namespace {
GemmArgs base_args(const StepParams& p) {
  GemmArgs g{};
  g.C = p.C; g.model = p.model; g.gamma = p.gamma; g.reg_coef = p.reg_coef; g.reg_norm = p.reg_norm;
  g.Cs = p.Cs; g.Ns = p.Ns; g.D = p.D;
  return g;
}
}  // namespace

// S = A . Bn^T  (+ TransE_l2 distance epilogue)
int umma_score(const LaunchCtx& c, const StepParams& p, const StepWs& w) {
  // operands arrive already split: k_prep writes A / Bn as TF32 hi/lo, k_loss writes V hi/lo
  CUtensorMap ah, al, bh, bl;
  const long long rowsA = p.B * (long long)slab_blocks(p.D), rowsB = p.Nn * (long long)slab_blocks(p.D);
  if (tc_make_map(&ah, w.Ahi, rowsA, 32, kTileM) || tc_make_map(&al, w.Alo, rowsA, 32, kTileM) ||
      tc_make_map(&bh, w.Bhi, rowsB, 32, kTileN) || tc_make_map(&bl, w.Blo, rowsB, 32, kTileN))
    return KGE_ERR_CUDA;
  GemmArgs g = base_args(p);
  g.mode = G_SCORE; g.M = p.Cs; g.N = p.Ns; g.K = p.D;
  g.a_nblk = slab_blocks(p.D); g.a_R = p.Cs; g.b_nblk = slab_blocks(p.D); g.b_R = p.Ns;
  g.out = w.S; g.out2 = w.V; g.a2 = w.a2; g.b2 = w.b2;
  return launch_gemm<G_SCORE>(c, ah, al, bh, bl, g);
}

// side_b == false: GA = V . Bn ; side_b == true: G_neg = V^T . A (+ epilogue), in place over Bn
int umma_grad(const LaunchCtx& c, const StepParams& p, const StepWs& w, bool side_b) {
  CUtensorMap ah, al, bh, bl;
  GemmArgs g = base_args(p);
  g.colsum = w.colsum;
  if (!side_b) {
    // A operand: V slabs [C][Ns/32][Cs][32]; B operand: Bn^T slabs [C][Ns/32][D][32]; K = j
    const long long rowsV = p.B * (long long)slab_blocks(p.Ns), rowsB = (long long)p.C * slab_blocks(p.Ns) * p.D;
    if (tc_make_map(&ah, w.Vhi, rowsV, 32, kTileM) || tc_make_map(&al, w.Vlo, rowsV, 32, kTileM) ||
        tc_make_map(&bh, w.BhiT, rowsB, 32, kTileN) || tc_make_map(&bl, w.BloT, rowsB, 32, kTileN))
      return KGE_ERR_CUDA;
    g.a_nblk = slab_blocks(p.Ns); g.a_R = p.Cs; g.b_nblk = slab_blocks(p.Ns); g.b_R = p.D;
    g.mode = G_GA; g.M = p.Cs; g.N = p.D; g.K = p.Ns; g.out = w.GA;
    return launch_gemm<G_GA>(c, ah, al, bh, bl, g);
  }
  // A operand: V^T slabs [C][Cs/32][Ns][32]; B operand: A^T slabs [C][Cs/32][D][32]; K = i
  const long long rowsV = (long long)p.C * slab_blocks(p.Cs) * p.Ns, rowsA = (long long)p.C * slab_blocks(p.Cs) * p.D;
  if (tc_make_map(&ah, w.VhiT, rowsV, 32, kTileM) || tc_make_map(&al, w.VloT, rowsV, 32, kTileM) ||
      tc_make_map(&bh, w.AhiT, rowsA, 32, kTileN) || tc_make_map(&bl, w.AloT, rowsA, 32, kTileN))
    return KGE_ERR_CUDA;
  g.a_nblk = slab_blocks(p.Cs); g.a_R = p.Ns; g.b_nblk = slab_blocks(p.Cs); g.b_R = p.D;
  g.mode = G_GB; g.M = p.Ns; g.N = p.D; g.K = p.Cs; g.out = w.Bn;
  return launch_gemm<G_GB>(c, ah, al, bh, bl, g);
}

}  // namespace kge
