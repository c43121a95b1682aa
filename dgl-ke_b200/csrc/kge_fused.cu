// kge_fused.cu -- the two contraction kernels of the fused step (wgmma / TMA / mbarrier, sm_90a):
//
//   k_fused<P>  rows = positives i, columns = negatives j:
//               S = A.Bn^T (tensor cores, accumulator in registers) -> loss / self-adversarial softmax / backward
//               coefficients V, written to shared memory in the order of wgmma's register A fragment -> GA = V.Bn
//               (tensor cores, V loaded per k-step as the REGISTER A operand, split into TF32 hi/lo) -> epilogue.
//               Replaces create_neg (score_fun.py:91-108,268-286,345-376,427-449), LossGenerator.get_total_loss
//               (loss.py:69-98) and the dL/da half of loss.backward().  The score matrix S never leaves the SM; V leaves
//               it once, as the transposed fp32 slab V^T[c][i / 32][j][i % 32] plus per-tile column sums sum_i V_ij,
//               for k_fused<N>; spare warps write both from the shared-memory copy while GEMM2 runs.
//   k_fused<N>  rows = negatives j:  G_neg = V^T.A - colsum*b + reg'(b), mean(G_neg^2)  (the dL/db half of
//               loss.backward() plus phase 1 of ExternalEmbedding.update for the negatives, tensor_models.py:316-328).
//               One pipelined GEMM over K = Cs: the V^T slab (written by k_fused<P>) as the register A operand and the
//               transposed A slabs (written by k_prep) from shared memory.
//
// Handing V over costs 4 B x C x Cs x Ns of HBM traffic each way (11.8 MB at 66 chunks of 200 x 200); recomputing it
// in the second orientation cost a whole K = D GEMM per chunk plus the loss epilogue, and an S accumulator that
// crowded the register file.  fp32 fidelity: operands are TF32 hi/lo pairs and every k-step issues hi*hi + hi*lo +
// lo*hi (3xTF32, fp32 accumulation).  B operands come from shared memory as hi/lo slabs.  An A operand is loaded as
// fp32 and split by the issuing thread into the register fragment (a_frag), so it crosses HBM once instead of twice --
// except next to a 256-column accumulator, where two fragment sets do not fit the register file (ptxas serialises or
// spills): those variants (kRegA false) read A as hi/lo slabs from shared memory, as the B operand.  wgmma reads TF32 operands from shared memory K-major only: GEMMs that contract over the rows of a matrix
// take its transposed slabs (kge_common.cuh:slabT_off).
//
// CTA = 384 threads: warpgroups 0 and 1 (warps 0-7) each own 64 rows of the 128-row tile -- MMA issue and epilogue on
// the accumulator fragment, a row lives in the 4 lanes of a quad; warp 8 TMA producer, warps 10-11 prefetch the next
// step's rows; in k_fused<P> warp 9 (and 10-11 when they do not prefetch) write the V hand-off.  Persistent over
// (chunk, 128-row tile) work items.
// Shared memory: one ring.  k_fused<P> (223 KB, 192 KB with prefetch slots) uses it as nS1 stages {X,Y_hi,Y_lo} for GEMM1, then as
// the V buffer followed by nS2 stages {Y^T_hi,Y^T_lo} for GEMM2, whose output is produced in chunks of NW columns;
// k_fused<N> (192 KB) as nS stages {V^T,A^T_hi,A^T_lo} of one output-column chunk of width NW.  X and V^T are fp32, or
// hi/lo pairs {X_hi,X_lo} / {V^T_hi,V^T_lo} in the 256-wide variants.
#include <cuda.h>
#include <cstdio>
#include <cstdlib>
#include <mutex>
#include "kge_common.cuh"
#include "kge_tc.cuh"

namespace kge {

using namespace tc;

namespace {

constexpr int kTileM = 128;
constexpr int kThreadsF = 384;                    // warps 0-7 MMA + epilogue (two warpgroups), 8 TMA producer, 10-11 prefetch
constexpr int kProducerWarp = 8;
constexpr int kHandoffWarp = 9;                    // k_fused<P>: first of the warps that write the V hand-off
constexpr int kMaxS1 = 4, kMaxS2 = 8;
constexpr int kMaxPf = 8;                          // row slots per prefetch warp
constexpr uint32_t kRingBytes = 192 * 1024;        // k_fused<N>
// k_fused<P>: the 227 KB a CTA may opt in to, less the 1 KB alignment slack of the ring, the kernel's static shared
// memory (mbarriers, |b|^2 of the chunk, the row scales: 2 KB as ptxas reports it) and 1 KB to spare
constexpr uint32_t kRingBytesP = 223 * 1024;
constexpr float kLog2e = 1.4426950408889634f;
constexpr float kLn2 = 0.6931471805599453f;

struct FusedArgs {
  int model, adversarial;
  float gamma, Tl2e, inv2B, uni;
  float reg_coef;
  int reg_norm;
  int C, Rx, Ry, D;      // rows per chunk on the lane side / on the contraction side of the last GEMM, row length
  int N1;                // P: wgmma N of GEMM1 (the kernel variant's width, >= Ry);  N: output-column chunk width
  int N2;                // P: output-column chunk width of GEMM2
  int nblkD;             // 32-column slab blocks of D
  int nS1, nS2;          // P: GEMM1 / GEMM2 stages;  N: nS1 stages
  uint32_t stage1Bytes, stage2Bytes;
  float* VT;             // [C][Cs/32][Ns][32] coefficients V_ij, fp32 (P writes, N reads) ...
  float *VhiT, *VloT;    //   ... or as TF32 hi/lo when k_fused<N> runs 256 columns wide (VhiT set: P writes these)
  float* colpart;        // [ceil(Cs/128)][C*Ns] per-tile column sums sum_i V_ij (TransE_l2; P writes, N reads)
  int ncolpart;          // N: number of those partials
  // mode P
  const float* x2;       // |a|^2 per positive (TransE_l2)
  const float* y2;       // |b|^2 per negative (TransE_l2)
  const float* pos;      // [B] positive scores
  const float* wt;       // [B] edge weights or null
  const float* wbar;     // [1] mean edge weight (with wt)
  float *gpos, *rowsum, *pl, *nl;
  float* dumpS;          // optional [C*Rx, Ry]: negative scores (kge_debug_read)
  float* dumpV;          // optional: P [C*Cs, Ns] and N [C*Ns, Cs] views of the backward coefficients (tests)
  // mode N
  const float *Xhi, *Xlo;  // slabs of the negatives' rows: b = hi + lo in the epilogue
  const long long* xids;   // mode N, one GPU: entity ids of the negatives -- b is then read from the table itself
  TableView xtab;          //   (one fp32 load instead of hi + lo; nothing updates the table before k_update)
  const float* xraw;       // mode N, sharded + staged: the negatives' rows as fp32 [C*Ns, D] (the previous step's prefetch)
  float* gsn;            // [C*Ns] mean(G_neg^2)
  float* out;            // P: GA [C*Cs, D]; N: G_neg [C*Ns, D]
  // next step's rows, copied by the two spare warps while this step's tiles are computed (sharded tables: the remote-row
  // latency of step k+1 hides behind the tensor-core work of step k).  Virtual row v of [nodes | negatives]; this launch
  // takes the v with v % 2 == pf_parity (the P and the N kernel split the list).
  int pf_slots;                    // row slots per warp (0 = no prefetch), carved from the ring behind the GEMM stages
  int pf_parity;
  int pf_lag;                      // stores between a slot's own store and its re-load (>= 1)
  uint32_t pf_off, pf_row_bytes;
  const long long* pf_node_ids;    // next batch's unique nodes
  const long long* pf_nU_dev;      // their count on the device, or null
  long long pf_nU, pf_nNeg;
  const long long* pf_neg_ids;
  float* pf_nc;                    // [nU, D] destination of the node rows (the next step's NC)
  float* pf_bn;                    // [nNeg, D] destination of the negative rows
};

// regulariser gradient in the epilogue: the default norm (3) inline, anything else out of line (code size: the
// epilogue is instruction-cache sensitive)
static __device__ __noinline__ float reg_grad_any(float b, int norm, float coef) { return reg_grad(b, norm, coef); }
__device__ __forceinline__ float reg_grad_fast(float b, int norm, float coef) {
  if (norm == 3) return 3.f * coef * fabsf(b) * b;
  return reg_grad_any(b, norm, coef);
}

__device__ __forceinline__ void epi_bar() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

// ================================ prefetch warps 10, 11 (both kernels) ================================
// Each warp streams table rows (peer memory when the table is sharded) through a few shared-memory slots into the
// next step's buffers: bulk load -> mbarrier -> bulk store, S slots per warp re-used round robin.  The loop is warp-uniform
// (one elected lane issues): the row ids arrive 32 at a time, one coalesced load per lane, and are handed out by shuffle
// -- a per-row dependent id load by a single lane costs more than the copy itself.
__device__ __forceinline__ void prefetch_rows(const FusedArgs& g, uint8_t* ring, uint64_t (*pf_full)[kMaxPf], int w, int lane) {
  const int S = g.pf_slots;
  const long long nU = g.pf_nU_dev ? *g.pf_nU_dev : g.pf_nU;
  const long long total = nU + g.pf_nNeg;
  const long long nhalf = total > g.pf_parity ? (total - g.pf_parity + 1) / 2 : 0;   // v = parity + 2 j < total
  const long long stride = 2ll * gridDim.x, j0 = 2ll * blockIdx.x + w;
  const long long n = j0 < nhalf ? (nhalf - j0 + stride - 1) / stride : 0;
  uint8_t* slots = ring + g.pf_off + (size_t)w * S * g.pf_row_bytes;
  auto vrow = [&](long long k) { return g.pf_parity + 2 * (j0 + k * stride); };
  auto fetch_ids = [&](long long kb) {            // ids of items kb .. kb+31, one per lane
    const long long k = kb + lane;
    if (k >= n) return 0ll;
    const long long v = vrow(k);
    return v < nU ? g.pf_node_ids[v] : g.pf_neg_ids[v - nU];
  };
  long long ids_lo = fetch_ids(0), ids_hi = fetch_ids(32);      // items [base, base+32) and [base+32, base+64)
  long long base = 0;
  auto load = [&](long long k) {                  // k in [base, base + 64)
    const int o = (int)(k - base);
    const long long id = __shfl_sync(0xffffffffu, o < 32 ? ids_lo : ids_hi, o & 31);
    const int s = (int)(k % S);
    if (elect_one()) {
      mbar_expect_tx(&pf_full[w][s], g.pf_row_bytes);
      bulk_g2s(slots + (size_t)s * g.pf_row_bytes, row_ptr(g.xtab, id), g.pf_row_bytes, &pf_full[w][s]);
    }
    __syncwarp();
  };
  for (long long k = 0; k < n && k < S; ++k) load(k);
  // A slot is re-loaded L stores after its own store was issued (S - L loads in flight).  L = 1 keeps the most loads in
  // flight, which is what matters when the rows are remote; a larger L (KGE_B200_PF_LAG) never waits on the copy
  // engine's queue for the newest store.
  const int L = g.pf_lag < S - 1 ? g.pf_lag : (S > 2 ? S - 2 : 1);
  for (long long k = 0; k < n; ++k) {
    const int s = (int)(k % S);
    mbar_wait(&pf_full[w][s], (uint32_t)((k / S) & 1));
    const long long v = vrow(k);
    float* dst = v < nU ? g.pf_nc + v * (long long)g.D : g.pf_bn + (v - nU) * (long long)g.D;
    const long long kr = k - L + S;                // the item that takes over the slot of item k - L
    const bool reload = k >= L && kr < n;
    // rotate the id window one batch early: the fresh batch is needed 32 items from now
    if (reload && kr >= base + 32) { base += 32; ids_lo = ids_hi; ids_hi = fetch_ids(base + 32); }
    if (elect_one()) {
      bulk_s2g(dst, slots + (size_t)s * g.pf_row_bytes, g.pf_row_bytes);
      bulk_commit();
      if (reload) { if (L == 3) bulk_wait_read<3>(); else if (L == 2) bulk_wait_read<2>(); else bulk_wait_read<1>(); }
    }
    __syncwarp();
    if (reload) load(kr);
  }
  if (elect_one()) bulk_wait_all();
  __syncwarp();
}

// A 256-wide accumulator leaves no room for register fragments: such variants use k_reg_a() false
__host__ __device__ constexpr bool k_reg_a(int n) { return n < 256; }

// one k-block of a GEMM with both operands in shared memory: KS k-steps of 8, each hi*hi + hi*lo + lo*hi, as one wgmma
// group.  A guard between the fence and the commit would make ptxas insert warpgroup arrives of its own, so callers
// switch over the k-step count.
template <int NW, int KS>
__device__ __forceinline__ void kblock_3xtf32(float (&acc)[NW / 2], uint64_t dXh, uint64_t dXl, uint64_t dYh, uint64_t dYl) {
  wgmma_fence();
#pragma unroll
  for (int ks = 0; ks < KS; ++ks) {
    const uint64_t o = (uint64_t)(ks * 2);     // K-major: +32 bytes per k-step inside the 128-byte swizzle span
    wgmma_ss<NW>(acc, dXh + o, dYh + o, 1u);
    wgmma_ss<NW>(acc, dXh + o, dYl + o, 1u);
    wgmma_ss<NW>(acc, dXl + o, dYh + o, 1u);
  }
  wgmma_commit();
}

__device__ __forceinline__ float lds_f32(uint32_t a) {
  float v;
  asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(a) : "memory");
  return v;
}

// The register A fragment of k-step ks from an fp32 stage of 128 rows x 32 floats (K-major, TMA 128-byte swizzle: the
// 16-byte chunk c of row r sits at chunk position c ^ (r & 7)), split into TF32 hi/lo.  Thread (g = lane / 4,
// q = lane % 4) of MMA warp w reads (r, k = 8 ks + q), (r + 8, q), (r, q + 4), (r + 8, q + 4) for r = 16 w + g, i.e.
// float q of chunk 2 ks (+1 for q + 4).  r and r + 8 share r & 7 = g, so each of the four loads reaches bank
// 4 ((2 ks [+1]) ^ g) + q: the 8 values of g give 8 distinct chunk positions and q the 4 words in each, so the 32 lanes
// hit 32 distinct banks.  `row` is the shared address of row r.
__device__ __forceinline__ void a_frag(uint32_t row, int ks, int g, int q, uint32_t (&ah)[4], uint32_t (&al)[4]) {
  const uint32_t c0 = row + (uint32_t)(((((2 * ks) ^ g) << 2) + q) << 2);
  const uint32_t c1 = row + (uint32_t)(((((2 * ks + 1) ^ g) << 2) + q) << 2);
  const float a[4] = {lds_f32(c0), lds_f32(c0 + 1024u), lds_f32(c1), lds_f32(c1 + 1024u)};
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    float hi, lo;
    split_tf32(a[r], hi, lo);
    ah[r] = __float_as_uint(hi); al[r] = __float_as_uint(lo);
  }
}

// one k-step hi*hi + hi*lo + lo*hi as one wgmma group, the A fragment in registers
template <int N>
__device__ __forceinline__ void kstep_rs(float (&acc)[N / 2], const uint32_t (&ah)[4], const uint32_t (&al)[4],
                                         uint64_t dYh, uint64_t dYl) {
  wgmma_fence();
  wgmma_rs<N>(acc, ah, dYh, 1u);
  wgmma_rs<N>(acc, ah, dYl, 1u);
  wgmma_rs<N>(acc, al, dYh, 1u);
  wgmma_commit();
}

// One k-block of KS k-steps of 8 whose A operand is an fp32 stage (a_frag) and whose B operand is a hi/lo pair of
// shared-memory slabs: one wgmma group per k-step, at most two in flight.  Two fragment sets alternate and a set is
// re-written only once the group that reads it has retired; every k-block but the last has 4 k-steps, so k-step ks
// always takes set ks & 1.  `release`: the previous k-block's stage, handed back once the first group of this one is
// issued and the previous one's last group has retired (its ld.shared reads are done before its wgmmas are issued).
// A guard between a fence and a commit would make ptxas insert warpgroup arrives of its own, so callers switch over the
// k-step count.
template <int N, int KS>
__device__ __forceinline__ void kblock_rs(float (&acc)[N / 2], uint32_t (&ah)[2][4], uint32_t (&al)[2][4], uint32_t row,
                                          int g, int q, uint64_t dYh, uint64_t dYl, uint64_t* release, int lane) {
#pragma unroll
  for (int ks = 0; ks < KS; ++ks) {
    a_frag(row, ks, g, q, ah[ks & 1], al[ks & 1]);
    const uint64_t o = (uint64_t)(ks * 2);     // K-major: +32 bytes per k-step inside the 128-byte swizzle span
    kstep_rs<N>(acc, ah[ks & 1], al[ks & 1], dYh + o, dYl + o);
    wgmma_wait<1>();                           // the previous k-step has retired: its fragment set is free
    reg_fence(ah[(ks + 1) & 1]); reg_fence(al[(ks + 1) & 1]);
    if (ks == 0 && release && lane == 0) mbar_arrive(release);
  }
}

// ================================ k_fused<P> ================================
// The coefficients V of the tile in shared memory, in the order of GEMM2's register A fragment: per MMA warp w and k-step
// j (8 columns), 32 lanes x 16 bytes = (row, k = q), (row + 8, q), (row, q + 4), (row + 8, q + 4) of lane 4 g + q, so a
// k-step is one 16-byte ld.shared per thread.  The lane's 16 bytes sit at position L ^ ((L >> 3) & 3): the fragment
// loads stay conflict-free (the 8 lanes of a quarter warp keep distinct positions mod 8, so they cover all 32 banks);
// the scalar stores from the accumulator fragment (32 lanes, 16 lane positions) and the hand-off warps' column reads
// (32 consecutive rows of one column) both reach 16 banks, so every bank at most twice.  Returns the float index.
template <int NV>
__device__ __forceinline__ int vsm_idx(int i, int k) {          // i: row of the tile (0..127), k: column (0..NV-1)
  const int g = i & 7, h = (i >> 3) & 1, kk = k & 7;
  const int L = 4 * g + (kk & 3);
  return (((i >> 4) * (NV / 8) + (k >> 3)) * 32 + (L ^ ((L >> 3) & 3))) * 4 + h + 2 * (kk >> 2);
}

// GEMM2 k-step j of one output chunk: the fragment from shared memory, split into TF32 hi/lo, hi*hi + hi*lo + lo*hi as one
// wgmma group.  Two fragment sets alternate (a set is re-written only once the group that reads it has retired).
template <int NW>
__device__ __forceinline__ void pos_kstep(float (&acc2)[NW / 2], uint32_t (&ah)[4], uint32_t (&al)[4], const float* vf,
                                          uint64_t dYh, uint64_t dYl) {
  const float4 v = *reinterpret_cast<const float4*>(vf);
  const float a[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    float hi, lo;
    split_tf32(a[r], hi, lo);
    ah[r] = __float_as_uint(hi); al[r] = __float_as_uint(lo);
  }
  kstep_rs<NW>(acc2, ah, al, dYh, dYl);
}

// this thread's first row inside the 128-row tile (16 per warp, lane / 4; the second is 8 further): read from %tid.x
// where it is needed rather than held across GEMM1 and the softmax passes, where every register not taken by the score
// accumulator is wanted and ptxas would spill it
__device__ __forceinline__ int tile_row() {
  uint32_t t;
  asm volatile("mov.u32 %0, %%tid.x;" : "=r"(t));
  return (int)((t >> 5) * 16 + ((t >> 2) & 7));
}

template <int NV, int NW>
__global__ void __launch_bounds__(kThreadsF, 1)
k_fused_pos(const __grid_constant__ CUtensorMap mX, const __grid_constant__ CUtensorMap mXl,   // mXl: !k_reg_a(NV) only
            const __grid_constant__ CUtensorMap mYh1, const __grid_constant__ CUtensorMap mYl1,
            const __grid_constant__ CUtensorMap mYh2, const __grid_constant__ CUtensorMap mYl2, FusedArgs g) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t full1[kMaxS1], empty1[kMaxS1], full2[kMaxS2], empty2[kMaxS2];
  __shared__ __align__(8) uint64_t vfree;           // the tile's V buffer is no longer read (MMA and hand-off warps)
  __shared__ __align__(8) uint64_t pf_full[2][kMaxPf];
  __shared__ __align__(16) float colA[NV];
  __shared__ float rsc[kTileM];                    // 1 / softmax denominator (or 1 / Ns) of each row of the tile

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  uint8_t* ring = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  float* vsm = reinterpret_cast<float*>(ring);      // V buffer: overlays the GEMM1 stages, ahead of the GEMM2 stages
  constexpr uint32_t vBytes = (uint32_t)NV * 512u;  // 8 warps x NV / 8 k-steps x 512 bytes
  uint8_t* ring2 = ring + vBytes;

  const int mtiles = (g.Rx + kTileM - 1) / kTileM;
  const int ntiles = g.C * mtiles;
  const int nkb1 = (g.D + 31) >> 5;
  const int nkb2 = (g.Ry + 31) >> 5;
  const int nchunks = (g.D + NW - 1) / NW;
  constexpr uint32_t yBytes1 = (uint32_t)NV * 128u;
  constexpr uint32_t xBytes1 = k_reg_a(NV) ? 16384u : 32768u;      // X as fp32, or as hi + lo
  constexpr uint32_t yBytes2 = (uint32_t)NW * 128u;
  const bool l2 = g.model == KGE_TRANSE_L2;
  // the hand-off warps: warp 9, and warps 10-11 when they do not prefetch; they meet the MMA warps at named barrier 2
  const int nhand = g.pf_slots > 0 ? 1 : 3;
  const uint32_t hand_bar_n = 256u + 32u * (uint32_t)nhand;

  if (threadIdx.x == 0) {
    for (int s = 0; s < kMaxS1; ++s) { mbar_init(&full1[s], 1); mbar_init(&empty1[s], 8); }
    for (int s = 0; s < kMaxS2; ++s) { mbar_init(&full2[s], 1); mbar_init(&empty2[s], 8); }
    mbar_init(&vfree, 8 + nhand);
    for (int s = 0; s < kMaxPf; ++s) { mbar_init(&pf_full[0][s], 1); mbar_init(&pf_full[1][s], 1); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  if (warp == kProducerWarp && lane == 0) {
    tma_prefetch_desc(&mX); if (!k_reg_a(NV)) tma_prefetch_desc(&mXl); tma_prefetch_desc(&mYh1); tma_prefetch_desc(&mYl1);
    tma_prefetch_desc(&mYh2); tma_prefetch_desc(&mYl2);
  }
  __syncthreads();

  // Roles.  The producer runs its loop with all 32 lanes (warp-uniform control flow) and one elected lane issues the
  // TMA ops.  Registers: the third warpgroup (producer, hand-off and prefetch warps) hands most of its share to the two
  // MMA warpgroups, which keep the score accumulator and then a GEMM2 accumulator chunk in registers.
  if (warp >= 8) {
  asm volatile("setmaxnreg.dec.sync.aligned.u32 56;");
  if (warp == kProducerWarp) {
    // ================================ TMA producer ================================
    uint32_t n1 = 0, n2 = 0, it = 0;   // stage fills issued so far (GEMM1 / GEMM2), tiles so far
    for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x, ++it) {
      const int c = tile / mtiles, m0 = (tile % mtiles) * kTileM;
      // the ring is about to be re-used with the GEMM1 layout: the previous tile's GEMM2 stages are consumed and its V
      // buffer is read (every MMA warp has retired its last GEMM2 group, every hand-off warp is done)
      if (it > 0) mbar_wait(&vfree, (it - 1) & 1);
      for (int kb = 0; kb < nkb1; ++kb, ++n1) {
        const uint32_t s = n1 % g.nS1;
        mbar_wait(&empty1[s], ((n1 / g.nS1) & 1) ^ 1);
        uint8_t* st = ring + (size_t)s * g.stage1Bytes;
        // slab layout: TMA row of (chunk c, 32-column block kb, row r) = (c * nblkD + kb) * R + r
        const int yx = (c * g.nblkD + kb) * g.Rx + m0;
        const int yy = (c * g.nblkD + kb) * g.Ry;
        if (elect_one()) {
          mbar_expect_tx(&full1[s], xBytes1 + 2u * yBytes1);
          tma_load_2d(st, &mX, &full1[s], 0, yx);
          if (!k_reg_a(NV)) tma_load_2d(st + 16384, &mXl, &full1[s], 0, yx);
          tma_load_2d(st + xBytes1, &mYh1, &full1[s], 0, yy);
          tma_load_2d(st + xBytes1 + yBytes1, &mYl1, &full1[s], 0, yy);
        }
        __syncwarp();
      }
      // GEMM2 stages overlay the GEMM1 stages: wait until the tensor core has consumed all of them
      for (uint32_t k = (n1 > (uint32_t)g.nS1 ? n1 - g.nS1 : 0); k < n1; ++k) mbar_wait(&empty1[k % g.nS1], (k / g.nS1) & 1);
      for (int ch = 0; ch < nchunks; ++ch) {
        for (int kb = 0; kb < nkb2; ++kb, ++n2) {
          const uint32_t s = n2 % g.nS2;
          mbar_wait(&empty2[s], ((n2 / g.nS2) & 1) ^ 1);
          uint8_t* st = ring2 + (size_t)s * g.stage2Bytes;
          // transposed slabs: TMA row of (chunk c, 32-row block kb of Y, column d) = (c * nblkRy + kb) * D + d
          const int yy = (c * nkb2 + kb) * g.D + ch * NW;
          if (elect_one()) {
            mbar_expect_tx(&full2[s], 2u * yBytes2);
            tma_load_2d(st, &mYh2, &full2[s], 0, yy);
            tma_load_2d(st + yBytes2, &mYl2, &full2[s], 0, yy);
          }
          __syncwarp();
        }
      }
    }
  } else if (warp - kHandoffWarp < nhand) {
    // ================================ V hand-off to k_fused<N> ================================
    // V_ij = coef_ij / den_i in the transposed fp32 slab V^T[c][i / 32][j][i % 32] (or its hi/lo pair, for a 256-wide
    // k_fused<N>): per column j and 32-row block, one lane per row, so every store is a whole 128-byte line; rows i >= Cs are not written (k_fused<N> never reads
    // them).  TransE_l2 also needs sum_i V_ij over the tile: each lane adds its rows of the blocks in order, then
    // a fixed butterfly over the lanes.  Both are read from the shared-memory copy while the MMA warps run GEMM2.
    const int hw = warp - kHandoffWarp;
    for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
      const int c = tile / mtiles, m0 = (tile % mtiles) * kTileM;
      const int rows = g.Rx - m0 < kTileM ? g.Rx - m0 : kTileM;
      const int nb = (rows + 31) >> 5;
      asm volatile("bar.sync 2, %0;" ::"r"(hand_bar_n) : "memory");     // V and rsc of the tile are in shared memory
      float* dst = g.colpart + (long long)(tile % mtiles) * g.C * g.Ry + (long long)c * g.Ry;
      for (int j = hw; j < g.Ry; j += nhand) {
        float s = 0.f;
        float v[kTileM / 32];                      // all blocks' loads issued before the first store
#pragma unroll
        for (int b = 0; b < kTileM / 32; ++b) {
          const int i = 32 * b + lane;
          v[b] = b < nb ? vsm[vsm_idx<NV>(i, j)] * rsc[i] : 0.f;
        }
#pragma unroll
        for (int b = 0; b < kTileM / 32; ++b) {
          const int i = 32 * b + lane;
          if (i < rows) {
            const long long o = slabT_off(c, g.Rx, g.Ry, m0 + i, j);
            if (g.VhiT) {
              float hi, lo;
              split_tf32(v[b], hi, lo);
              g.VhiT[o] = hi; g.VloT[o] = lo;
            } else {
              g.VT[o] = v[b];
            }
          }
          s += v[b];
        }
        if (l2) {
#pragma unroll
          for (int x = 16; x >= 1; x >>= 1) s += __shfl_xor_sync(0xffffffffu, s, x);
          if (lane == 0) dst[j] = s;
        }
      }
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");     // the next tile's TMA writes over the buffer
      __syncwarp();
      if (lane == 0) mbar_arrive(&vfree);
    }
  } else if (warp >= 10 && g.pf_slots > 0) {
    prefetch_rows(g, ring, pf_full, warp - 10, lane);
  }
  } else {
    // ================================ MMA + epilogue warps 0..7 ================================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 224;");
    const int q = lane & 3;
    const int et = threadIdx.x;                   // 0..255
    uint32_t n1 = 0, n2 = 0;
    for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
      const int c = tile / mtiles, m0 = (tile % mtiles) * kTileM;
      epi_bar();                                  // everybody is done with the previous tile's shared constants
      for (int y = et; y < NV; y += 256) {
        const bool ok = y < g.Ry;
        colA[y] = (l2 && ok) ? g.y2[(long long)c * g.Ry + y] : 0.f;
      }
      epi_bar();
      float rscal[2];                             // 1 / softmax denominator (or 1 / Ns) of the two rows
      {
      float acc[NV / 2];                          // S -> V: rows rloc (+8), columns 8 j + 2 q + {0, 1}
      // ---- GEMM1: S = X . Y^T, K = D; X (fp32) as the register A operand ----
#pragma unroll
      for (int i = 0; i < NV / 2; ++i) acc[i] = 0.f;
      if constexpr (k_reg_a(NV)) {
        uint32_t ah[2][4], al[2][4];
        const int g8 = (lane >> 2);
        for (int kb = 0; kb < nkb1; ++kb, ++n1) {
          const uint32_t s = n1 % g.nS1;
          mbar_wait(&full1[s], (n1 / g.nS1) & 1);
          const uint32_t st = smem_u32(ring + (size_t)s * g.stage1Bytes);
          const uint32_t xrow = st + (uint32_t)(16 * warp + g8) * 128u;
          const uint64_t dYh = make_desc(st + xBytes1), dYl = make_desc(st + xBytes1 + yBytes1);
          const int kleft = g.D - kb * 32;
          const int ksteps = kleft >= 32 ? 4 : (kleft >> 3);
          uint64_t* rel = kb > 0 ? &empty1[(n1 - 1) % g.nS1] : nullptr;
          switch (ksteps) {
            case 4: kblock_rs<NV, 4>(acc, ah, al, xrow, g8, q, dYh, dYl, rel, lane); break;
            case 3: kblock_rs<NV, 3>(acc, ah, al, xrow, g8, q, dYh, dYl, rel, lane); break;
            case 2: kblock_rs<NV, 2>(acc, ah, al, xrow, g8, q, dYh, dYl, rel, lane); break;
            default: kblock_rs<NV, 1>(acc, ah, al, xrow, g8, q, dYh, dYl, rel, lane); break;
          }
        }
        wgmma_wait<0>();
        reg_fence(ah[0]); reg_fence(ah[1]); reg_fence(al[0]); reg_fence(al[1]);
      } else {
        const int wg = warp >> 2;
        for (int kb = 0; kb < nkb1; ++kb, ++n1) {
          const uint32_t s = n1 % g.nS1;
          mbar_wait(&full1[s], (n1 / g.nS1) & 1);
          const uint32_t st = smem_u32(ring + (size_t)s * g.stage1Bytes);
          const uint64_t dXh = make_desc(st + wg * 8192u), dXl = make_desc(st + 16384u + wg * 8192u);
          const uint64_t dYh = make_desc(st + xBytes1), dYl = make_desc(st + xBytes1 + yBytes1);
          const int kleft = g.D - kb * 32;
          const int ksteps = kleft >= 32 ? 4 : (kleft >> 3);
          switch (ksteps) {
            case 4: kblock_3xtf32<NV, 4>(acc, dXh, dXl, dYh, dYl); break;
            case 3: kblock_3xtf32<NV, 3>(acc, dXh, dXl, dYh, dYl); break;
            case 2: kblock_3xtf32<NV, 2>(acc, dXh, dXl, dYh, dYl); break;
            default: kblock_3xtf32<NV, 1>(acc, dXh, dXl, dYh, dYl); break;
          }
          if (kb > 0) {
            wgmma_wait<1>();                           // the previous k-block has retired: its stage is free
            if (lane == 0) mbar_arrive(&empty1[(n1 - 1) % g.nS1]);
          }
        }
        wgmma_wait<0>();
      }
      if (lane == 0) mbar_arrive(&empty1[(n1 - 1) % g.nS1]);
      reg_fence(acc);
      epi_bar();                                  // both warpgroups' GEMM1 has retired: the V buffer may overwrite the stages
      const int rloc = tile_row();                // this thread's rows inside the tile: rloc, rloc + 8

      // ---- S -> V, two rows per thread; a row's statistics are reduced over the 4 lanes of its quad ----
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int m = m0 + rloc + 8 * h;
        const bool row_ok = m < g.Rx;
        const long long gx = (long long)c * g.Rx + (row_ok ? m : 0);
        const float x2v = (l2 && row_ok) ? g.x2[gx] : 0.f;
        const float w_i = (g.wt && row_ok) ? g.wt[gx] : 1.f;
        const float kw = w_i * g.inv2B;
        // ---- pass A: scores (distance epilogue for TransE_l2), running max ----
        float mxl = -INFINITY;
        if (g.adversarial || g.dumpS) {
#pragma unroll
          for (int j = 0; j < NV / 8; ++j) {
            float sv[2];
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int col = 8 * j + 2 * q + e;
              float s = acc[4 * j + 2 * h + e];
              if (l2) {
                // batched_l2_dist (score_fun.py:26-34): (|b|^2 - 2 a.b) + |a|^2, clamp 1e-30, sqrt
                const float sqc = fmaxf(fmaf(-2.f, s, colA[col]) + x2v, 1e-30f);
                s = g.gamma - sqc * rsqrta(sqc);
              }
              sv[e] = s;
              if (col < g.Ry) mxl = fmaxf(mxl, s * g.Tl2e);
            }
            if (g.dumpS && row_ok && 8 * j + 2 * q < g.Ry)
              *reinterpret_cast<float2*>(g.dumpS + gx * g.Ry + 8 * j + 2 * q) = make_float2(sv[0], sv[1]);
          }
        }
        if (g.adversarial) {
          mxl = fmaxf(mxl, __shfl_xor_sync(0xffffffffu, mxl, 1));
          mxl = fmaxf(mxl, __shfl_xor_sync(0xffffffffu, mxl, 2));
        } else {
          mxl = 0.f;
        }
        // ---- pass C: softmax numerators, loss terms and (unnormalised) backward coefficients, which go to the V
        //      buffer.  The 1/denominator of the row is a per-row scalar: it is applied to the loss sums here, to the
        //      hand-off by the hand-off warps and to the row of GA in the GEMM2 epilogue. ----
        float nls = 0.f, rs = 0.f, den = 0.f;
#pragma unroll
        for (int j = 0; j < NV / 8; ++j) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int col = 8 * j + 2 * q + e;
            float s = acc[4 * j + 2 * h + e], rinv = 1.f;
            if (l2) {
              const float sq = fmaf(-2.f, s, colA[col]) + x2v;
              const float sqc = fmaxf(sq, 1e-30f);
              const float r = rsqrta(sqc);
              s = g.gamma - sqc * r;
              rinv = (sq > 1e-30f) ? r : 0.f;        // clamped distance: zero gradient (clamp_min_), dist ~ 0
            }
            const float pe = g.adversarial ? ex2a(fmaf(s, g.Tl2e, -mxl)) : 1.f;
            const float t = ex2a(-fabsf(s) * kLog2e);
            const float u = 1.f + t;
            const float r1 = rcpa(u);
            const float sig = (s >= 0.f) ? r1 : t * r1;                     // sigmoid(s)
            const float sp = fmaf(kLn2, lg2a(u), fmaxf(s, 0.f));            // -logsigmoid(-s)
            const bool ok = row_ok && (col < g.Ry);
            const float coef = ok ? pe * sig * kw * rinv : 0.f;              // dL/dneg_ij (/ dist) * denominator
            if (ok) { nls = fmaf(pe, sp, nls); den += pe; }
            rs += coef;
            vsm[vsm_idx<NV>(rloc + 8 * h, col)] = coef;
          }
        }
        den += __shfl_xor_sync(0xffffffffu, den, 1); den += __shfl_xor_sync(0xffffffffu, den, 2);
        nls += __shfl_xor_sync(0xffffffffu, nls, 1); nls += __shfl_xor_sync(0xffffffffu, nls, 2);
        rs += __shfl_xor_sync(0xffffffffu, rs, 1); rs += __shfl_xor_sync(0xffffffffu, rs, 2);
        const float rscale = g.adversarial ? (row_ok ? 1.f / den : 0.f) : g.uni;
        rscal[h] = rscale;
        if (g.dumpV && row_ok) {        // test hook: the dump shows the normalised coefficients (each thread's own)
          for (int j = 0; j < NV / 8; ++j)
            if (8 * j + 2 * q < g.Ry)
              *reinterpret_cast<float2*>(g.dumpV + gx * g.Ry + 8 * j + 2 * q) =
                  make_float2(vsm[vsm_idx<NV>(rloc + 8 * h, 8 * j + 2 * q)] * rscale,
                              vsm[vsm_idx<NV>(rloc + 8 * h, 8 * j + 2 * q + 1)] * rscale);
        }
        if (q == 0 && row_ok) {
          const float ps = g.pos[gx];
          const float wb = g.wt ? *g.wbar : 1.f;        // loss.py:75,82: [B] * [B,1] -> mean(pl) * mean(w)
          g.pl[gx] = softplusf(-ps);
          g.nl[gx] = nls * rscale * w_i;
          g.gpos[gx] = -sigmoidf(-ps) * wb * g.inv2B;
          if (l2) g.rowsum[gx] = rs * rscale;
        }
      }
      if (q == 0) { rsc[rloc] = rscal[0]; rsc[rloc + 8] = rscal[1]; }
      }
      // the hand-off warps may read the tile's V and row scales; this warp reads back only its own rows
      asm volatile("bar.arrive 2, %0;" ::"r"(hand_bar_n) : "memory");
      __syncwarp();

      // ---- GEMM2: GA[:, chunk] = V . Bn[:, chunk], K = Ns, A operand from the V buffer; epilogue per NW-column chunk.
      //      One wgmma group per k-step, at most two in flight: a stage is released once the group of the next
      //      k-block's first k-step has been issued and its own last group has retired. ----
      const float* vw = vsm + ((warp * (NV / 8)) * 32 + (lane ^ ((lane >> 3) & 3))) * 4;
      const int rloc = tile_row();
      for (int ch = 0; ch < nchunks; ++ch) {
        const int d0 = ch * NW;
        float acc2[NW / 2];
#pragma unroll
        for (int i = 0; i < NW / 2; ++i) acc2[i] = 0.f;
        uint32_t ah[2][4], al[2][4];
#pragma unroll 1
        for (int kb = 0; kb < nkb2; ++kb) {
          const uint32_t s = n2 % g.nS2;
          mbar_wait(&full2[s], (n2 / g.nS2) & 1);
          const uint32_t st = smem_u32(ring2 + (size_t)s * g.stage2Bytes);
          const uint64_t dYh = make_desc(st), dYl = make_desc(st + yBytes2);
          const int kleft = g.Ry - kb * 32;
          const int ksteps = kleft >= 32 ? 4 : (kleft >> 3);
#pragma unroll
          for (int ks = 0; ks < 4; ++ks) {
            const int j = kb * 4 + ks;
            if (ks < ksteps) {
              const uint64_t o = (uint64_t)(ks * 2);
              pos_kstep<NW>(acc2, ah[j & 1], al[j & 1], vw + j * 128, dYh + o, dYl + o);
              if (j > 0) {
                wgmma_wait<1>();                        // k-step j - 1 has retired: its fragment set is free
                reg_fence(ah[(j - 1) & 1]); reg_fence(al[(j - 1) & 1]);
                if (ks == 0 && lane == 0) mbar_arrive(&empty2[(n2 - 1) % g.nS2]);   // ... and so has k-block kb - 1
              }
            }
          }
          ++n2;
        }
        wgmma_wait<0>();
        reg_fence(ah[0]); reg_fence(ah[1]); reg_fence(al[0]); reg_fence(al[1]);
        if (lane == 0) mbar_arrive(&empty2[(n2 - 1) % g.nS2]);
        reg_fence(acc2);
        // chunk epilogue from the fragment: rows rloc (+8), columns d0 + 8 j + 2 q + {0, 1}
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int m = m0 + rloc + 8 * h;
          if (m >= g.Rx) continue;
          float* orow = g.out + ((long long)c * g.Rx + m) * (long long)g.D;
#pragma unroll
          for (int j = 0; j < NW / 8; ++j) {
            const int k = d0 + 8 * j + 2 * q;
            if (k >= g.D) continue;
            // 1 / softmax denominator of the row
            *reinterpret_cast<float2*>(orow + k) = make_float2(acc2[4 * j + 2 * h] * rscal[h], acc2[4 * j + 2 * h + 1] * rscal[h]);
          }
        }
      }
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");     // the next tile's TMA writes over the V buffer
      __syncwarp();
      if (lane == 0) mbar_arrive(&vfree);
    }
  }
}

// ================================ k_fused<N> ================================
// float2 loads of b in flight per thread in the k_fused<N> chunk epilogue (32 registers next to the accumulator)
constexpr int kNegEpiLoads = 16;

// G_neg[c][j, d0 : d0 + NW] = sum_i V^T[j, i] A[i, d0 : d0 + NW] for one 128-row tile of negatives j and one output
// chunk of NW columns per pass over K = Cs; the stages carry the tile's V^T k-block and the chunk's A^T k-block.
// FLAT: the epilogue reads each negative's b as one fp32 row (the table, or the rows the previous step staged);
// otherwise as hi + lo from the slabs.  The source is fixed per launch, so the column loop never branches on it.
template <int NW, bool FLAT>
__global__ void __launch_bounds__(kThreadsF, 1)
k_fused_neg(const __grid_constant__ CUtensorMap mV, const __grid_constant__ CUtensorMap mVl,   // mVl: !k_reg_a(NW) only
            const __grid_constant__ CUtensorMap mAh, const __grid_constant__ CUtensorMap mAl, FusedArgs g) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t full[kMaxS1], empty[kMaxS1];
  __shared__ __align__(8) uint64_t pf_full[2][kMaxPf];

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  uint8_t* ring = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);

  const int mtiles = (g.Rx + kTileM - 1) / kTileM;
  const int ntiles = g.C * mtiles;
  const int nkb = (g.Ry + 31) >> 5;               // k-blocks of K = Cs
  const int nch = (g.D + NW - 1) / NW;
  constexpr uint32_t aBytes = (uint32_t)kTileM * 128u;
  constexpr uint32_t bBytes = (uint32_t)NW * 128u;
  constexpr uint32_t vBytes = k_reg_a(NW) ? aBytes : 2u * aBytes;     // V^T as fp32, or as hi + lo
  const bool l2 = g.model == KGE_TRANSE_L2;

  if (threadIdx.x == 0) {
    for (int s = 0; s < kMaxS1; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 8); }
    for (int s = 0; s < kMaxPf; ++s) { mbar_init(&pf_full[0][s], 1); mbar_init(&pf_full[1][s], 1); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  if (warp == kProducerWarp && lane == 0) {
    tma_prefetch_desc(&mV); if (!k_reg_a(NW)) tma_prefetch_desc(&mVl); tma_prefetch_desc(&mAh); tma_prefetch_desc(&mAl);
  }
  __syncthreads();

  if (warp >= 8) {
  asm volatile("setmaxnreg.dec.sync.aligned.u32 56;");
  if (warp == kProducerWarp) {
    // ================================ TMA producer ================================
    uint32_t n = 0;
    for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
      const int c = tile / mtiles, m0 = (tile % mtiles) * kTileM;
      for (int ch = 0; ch < nch; ++ch) {
        for (int kb = 0; kb < nkb; ++kb, ++n) {
          const uint32_t s = n % g.nS1;
          mbar_wait(&empty[s], ((n / g.nS1) & 1) ^ 1);
          uint8_t* st = ring + (size_t)s * g.stage1Bytes;
          // transposed slabs: TMA row of (chunk c, 32-row block kb, column) = (c * nkb + kb) * columns + column
          const int yv = (c * nkb + kb) * g.Rx + m0;
          const int ya = (c * nkb + kb) * g.D + ch * NW;
          if (elect_one()) {
            mbar_expect_tx(&full[s], vBytes + 2u * bBytes);
            tma_load_2d(st, &mV, &full[s], 0, yv);
            if (!k_reg_a(NW)) tma_load_2d(st + aBytes, &mVl, &full[s], 0, yv);
            tma_load_2d(st + vBytes, &mAh, &full[s], 0, ya);
            tma_load_2d(st + vBytes + bBytes, &mAl, &full[s], 0, ya);
          }
          __syncwarp();
        }
      }
    }
  } else if (warp >= 10 && g.pf_slots > 0) {
    prefetch_rows(g, ring, pf_full, warp - 10, lane);
  }
  } else {
    // ================================ MMA + epilogue warps 0..7 ================================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 224;");
    const int wg = warp >> 2, q = lane & 3;
    const int et = threadIdx.x;                   // 0..255
    const int rloc = wg * 64 + (warp & 3) * 16 + (lane >> 2);      // this thread's rows inside the tile: rloc, rloc + 8
    uint32_t n = 0;
    for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
      const int c = tile / mtiles, m0 = (tile % mtiles) * kTileM;
      if (g.dumpV) {
        // test hook: the coefficients this tile reads, [C*Ns, Cs], as the MMAs see them (hi + lo of the split)
        for (int e = et; e < kTileM * g.Ry; e += 256) {
          const int j = m0 + e / g.Ry, i = e % g.Ry;
          if (j >= g.Rx) break;
          const long long o = slabT_off(c, g.Ry, g.Rx, i, j);
          float hi, lo;
          if (k_reg_a(NW)) split_tf32(g.VT[o], hi, lo);
          else { hi = g.VhiT[o]; lo = g.VloT[o]; }
          g.dumpV[((long long)c * g.Rx + j) * g.Ry + i] = hi + lo;
        }
      }
      // sum_i V_ij of this thread's two rows: the per-tile partials of k_fused<P>, added in a fixed order
      float cs[2] = {0.f, 0.f};
      if (l2) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int m = m0 + rloc + 8 * h;
          if (m >= g.Rx) continue;
          const float* p = g.colpart + (long long)c * g.Rx + m;
          for (int t = 0; t < g.ncolpart; ++t) cs[h] += p[(long long)t * g.C * g.Rx];
        }
      }
      // where this thread's two rows of b start: the row itself (FLAT) or its offset in the slabs, once per tile.  Nothing
      // writes these sources while the kernel runs (the prefetch warps stage into the other of two buffers), so they are
      // read through the non-coherent path.
      bool rok[2];
      const float* brow[2] = {nullptr, nullptr};
      long long boff[2] = {0, 0};
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int m = m0 + rloc + 8 * h;
        rok[h] = m < g.Rx;
        if (!rok[h]) continue;
        const long long gx = (long long)c * g.Rx + m;
        if (FLAT) brow[h] = g.xraw ? g.xraw + gx * (long long)g.D : row_ptr(g.xtab, g.xids[gx]);
        else boff[h] = slab_off(c, g.nblkD, g.Rx, m, 0);
      }
      const long long blk = 32ll * g.Rx;          // slab stride between 32-column blocks of a row
      // b of column pairs j0 .. j0 + NB - 1 of row h into registers, all of them before any store of the batch: a row
      // waits for at most ceil(NJ / NB) load round trips per chunk instead of one per column pair
      constexpr int NJ = NW / 8;                  // column pairs per row and chunk
      constexpr int NB = FLAT ? kNegEpiLoads : kNegEpiLoads / 2;
      // the first batch of row 0 goes out before the last k-block's MMAs retire, except on the 256-wide slab path, where
      // holding it next to the 128-register accumulator makes ptxas spill
      constexpr bool early = FLAT || NW < 256;
      float2 bh[NB], bl[NB];
      auto load_b = [&](int h, int d0, int j0) {
#pragma unroll
        for (int jj = 0; jj < NB; ++jj) {
          const int k = d0 + 8 * (j0 + jj) + 2 * q;
          if (j0 + jj >= NJ || k >= g.D || !rok[h]) continue;
          if (FLAT) {
            bh[jj] = __ldg(reinterpret_cast<const float2*>(brow[h] + k));
          } else {
            const long long so = boff[h] + (k >> 5) * blk + (k & 31);
            bh[jj] = __ldg(reinterpret_cast<const float2*>(g.Xhi + so));
            bl[jj] = __ldg(reinterpret_cast<const float2*>(g.Xlo + so));
          }
        }
      };
      float gsq[2] = {0.f, 0.f};
      for (int ch = 0; ch < nch; ++ch) {
        const int d0 = ch * NW;
        float acc[NW / 2];                        // rows rloc (+8), columns d0 + 8 j + 2 q + {0, 1}
#pragma unroll
        for (int i = 0; i < NW / 2; ++i) acc[i] = 0.f;
        if constexpr (k_reg_a(NW)) {
          uint32_t ah[2][4], al[2][4];
          for (int kb = 0; kb < nkb; ++kb, ++n) {
            const uint32_t s = n % g.nS1;
            mbar_wait(&full[s], (n / g.nS1) & 1);
            const uint32_t st = smem_u32(ring + (size_t)s * g.stage1Bytes);
            const uint32_t vrow = st + (uint32_t)(16 * warp + (lane >> 2)) * 128u;
            const uint64_t dAh = make_desc(st + vBytes), dAl = make_desc(st + vBytes + bBytes);
            // K = Cs is a multiple of 8: the partial last block runs its whole k-steps and never reads the padding
            const int kleft = g.Ry - kb * 32;
            const int ksteps = kleft >= 32 ? 4 : (kleft >> 3);
            uint64_t* rel = kb > 0 ? &empty[(n - 1) % g.nS1] : nullptr;
            switch (ksteps) {
              case 4: kblock_rs<NW, 4>(acc, ah, al, vrow, lane >> 2, q, dAh, dAl, rel, lane); break;
              case 3: kblock_rs<NW, 3>(acc, ah, al, vrow, lane >> 2, q, dAh, dAl, rel, lane); break;
              case 2: kblock_rs<NW, 2>(acc, ah, al, vrow, lane >> 2, q, dAh, dAl, rel, lane); break;
              default: kblock_rs<NW, 1>(acc, ah, al, vrow, lane >> 2, q, dAh, dAl, rel, lane); break;
            }
          }
          if (early) load_b(0, d0, 0);
          wgmma_wait<0>();
          reg_fence(ah[0]); reg_fence(ah[1]); reg_fence(al[0]); reg_fence(al[1]);
        } else {
          for (int kb = 0; kb < nkb; ++kb, ++n) {
            const uint32_t s = n % g.nS1;
            mbar_wait(&full[s], (n / g.nS1) & 1);
            const uint32_t st = smem_u32(ring + (size_t)s * g.stage1Bytes);
            const uint64_t dVh = make_desc(st + wg * 8192u), dVl = make_desc(st + aBytes + wg * 8192u);
            const uint64_t dAh = make_desc(st + vBytes), dAl = make_desc(st + vBytes + bBytes);
            const int kleft = g.Ry - kb * 32;
            const int ksteps = kleft >= 32 ? 4 : (kleft >> 3);
            switch (ksteps) {
              case 4: kblock_3xtf32<NW, 4>(acc, dVh, dVl, dAh, dAl); break;
              case 3: kblock_3xtf32<NW, 3>(acc, dVh, dVl, dAh, dAl); break;
              case 2: kblock_3xtf32<NW, 2>(acc, dVh, dVl, dAh, dAl); break;
              default: kblock_3xtf32<NW, 1>(acc, dVh, dVl, dAh, dAl); break;
            }
            if (kb > 0) {
              wgmma_wait<1>();                         // the previous k-block has retired: its stage is free
              if (lane == 0) mbar_arrive(&empty[(n - 1) % g.nS1]);
            }
          }
          if (early) load_b(0, d0, 0);
          wgmma_wait<0>();
        }
        if (lane == 0) mbar_arrive(&empty[(n - 1) % g.nS1]);
        reg_fence(acc);
        // chunk epilogue from the fragment (the producer is already filling the next chunk's stages)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          if (!rok[h]) continue;
          float* orow = g.out + ((long long)c * g.Rx + m0 + rloc + 8 * h) * (long long)g.D;
#pragma unroll
          for (int j0 = 0; j0 < NJ; j0 += NB) {
            if (!early || h > 0 || j0 > 0) load_b(h, d0, j0);
#pragma unroll
            for (int jj = 0; jj < NB; ++jj) {
              const int j = j0 + jj;
              const int k = d0 + 8 * j + 2 * q;
              if (j >= NJ || k >= g.D) continue;
              float o0 = acc[4 * j + 2 * h], o1 = acc[4 * j + 2 * h + 1];
              const float2 b = FLAT ? bh[jj] : make_float2(bh[jj].x + bl[jj].x, bh[jj].y + bl[jj].y);
              if (l2) { o0 = fmaf(b.x, -cs[h], o0); o1 = fmaf(b.y, -cs[h], o1); }   // sum_i V_ij a_i - (sum_i V_ij) b_j
              o0 += reg_grad_fast(b.x, g.reg_norm, g.reg_coef);
              o1 += reg_grad_fast(b.y, g.reg_norm, g.reg_coef);
              gsq[h] += o0 * o0 + o1 * o1;
              *reinterpret_cast<float2*>(orow + k) = make_float2(o0, o1);
            }
          }
        }
      }
      // mean(G_neg^2) per row: the 4 lanes that share a row
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float v = gsq[h];
        v += __shfl_xor_sync(0xffffffffu, v, 1);
        v += __shfl_xor_sync(0xffffffffu, v, 2);
        const int m = m0 + rloc + 8 * h;
        if (q == 0 && m < g.Rx) g.gsn[(long long)c * g.Rx + m] = v / (float)g.D;
      }
    }
  }
}

}  // namespace

// The fused kernel keeps a whole row of the chunk's score matrix in the accumulator registers of one warpgroup
// (columns / 2 registers per thread): at most 240 columns.
// Its operands are those of the wgmma engine, and its epilogue is the plain (non-pairwise, unmasked) Logsigmoid criterion.
bool fused_supported(const StepParams& p) {
  return umma_supported(p) && !p.hinge && !p.pairwise && !p.neg_deg && p.Cs <= 240 && p.Ns <= 240;
}

// mode 0 (P): S = A.Bn^T -> loss, coefficients V -> GA, V^T slabs;  mode 1 (N): G_neg = V^T.A (+ mean square)
namespace {
// GEMM stage geometry of one mode + what the ring leaves for prefetch row slots.  A GEMM1 / k_fused<N> stage holds its
// A operand (kTileM x 128 B) once, as fp32, or as hi + lo in the 256-wide variants; layouts with prefetch slots are
// sized as if it always took a hi and a lo copy, so that their stage and slot counts do not depend on that.
constexpr uint32_t kLoBytes = (uint32_t)kTileM * 128u;
uint32_t stage1_bytes(int n) { return (k_reg_a(n) ? 1u : 2u) * kLoBytes + 2u * (uint32_t)n * 128u; }
struct Geometry { int Rx, Ry, N1, N2, nS1, nS2, pf_slots; uint32_t ringBytes, stage1Bytes, stage2Bytes, pf_off; bool ok; };

// k_fused<N>: the output-column chunk NW.  A pass over K streams the tile's V^T (128 rows) and the chunk's A^T (NW rows),
// 128 B per row and k-block, so a CTA streams nch * (128 + NW) rows per k-block for nch = ceil(D / NW) chunks: the
// width with the fewest is taken (d = 400: 2 x 200 -> 656 rows, against 768 for 2 x 256 and 1024 for 4 x 128).  A
// 256-wide stage (96 KB) fills the ring twice over, so it is not offered when prefetch slots are wanted.  Rows streamed
// decide, not ring depth: at d = 400, 2 stages of 2 x 200 beat 3 stages of 4 x 128 by 15 us per step on an H100.
int neg_chunk_width(int D, bool want_prefetch) {
  static const int widths[] = {64, 128, 200, 256};
  int best = 0;
  long long best_rows = 0;
  for (int w : widths) {
    if (w == 256 && want_prefetch) continue;
    const long long rows = (long long)((D + w - 1) / w) * (kTileM + w);
    if (!best || rows < best_rows) { best = w; best_rows = rows; }
  }
  return best;
}

Geometry geometry(const StepParams& p, int mode, bool want_prefetch) {
  Geometry q{};
  const uint32_t row = (uint32_t)p.D * 4u;
  if (mode == 1) {
    q.Rx = p.Ns; q.Ry = p.Cs;
    q.ringBytes = kRingBytes;
    q.N1 = neg_chunk_width(p.D, want_prefetch);
    q.stage1Bytes = stage1_bytes(q.N1);
    q.nS1 = (int)(kRingBytes / q.stage1Bytes); if (q.nS1 > kMaxS1) q.nS1 = kMaxS1;
    q.ok = q.nS1 >= 2;
    if (q.ok && want_prefetch) {
      // the GEMM gives up stages (never below 2) until both prefetch warps have kMaxPf row slots
      const uint32_t fp = stage1_bytes(q.N1) + (k_reg_a(q.N1) ? kLoBytes : 0u);
      int nS = (int)(kRingBytes / fp); if (nS > kMaxS1) nS = kMaxS1;
      while (nS > 2 && kRingBytes - (uint32_t)nS * fp < 2u * kMaxPf * row) --nS;
      const uint32_t used = (uint32_t)nS * fp;
      int slots = (int)((kRingBytes - used) / (2u * row));
      if (slots > kMaxPf) slots = kMaxPf;
      if (slots >= 2 && nS >= 2) { q.pf_slots = slots; q.nS1 = nS; q.pf_off = used; }
    }
    return q;
  }
  q.Rx = p.Cs; q.Ry = p.Ns;
  // wgmma's N is part of the instruction: the kernel is instantiated for these widths
  q.N1 = q.Ry <= 64 ? 64 : (q.Ry <= 128 ? 128 : (q.Ry <= 208 ? 208 : 256));
  // With prefetch slots the ring keeps the 192 KB they were carved from before the V buffer: whether the next step's
  // rows can be staged, and in how many slots, does not depend on the GEMM2 layout.  Without them it takes what a CTA
  // may opt in to.
  const uint32_t ring = want_prefetch ? kRingBytes : kRingBytesP;
  q.ringBytes = ring;
  q.stage1Bytes = stage1_bytes(q.N1);
  const uint32_t fp1 = (want_prefetch && k_reg_a(q.N1)) ? q.stage1Bytes + kLoBytes : q.stage1Bytes;
  int nS1 = (int)(ring / fp1); if (nS1 > kMaxS1) nS1 = kMaxS1;
  if (nS1 < 2) return q;
  // GEMM2 needs the V buffer (N1 / 8 k-steps x 512 B per MMA warp) ahead of its stages.  Its output-column chunk NW:
  // a chunk streams NW rows of Bn^T per k-block and issues NW columns of MMAs, so ceil(D / NW) * NW should be least
  // (d = 400: 2 x 200 = 400 against 4 x 128 = 512; d = 800: 4 x 200 against 7 x 128 = 896), 128 on a tie.  256 never
  // does better than 128.  A width is taken if the ring holds the buffer and 2 of its stages and, when prefetch slots
  // are wanted, leaves at least 2 of them; otherwise the next width, and prefetch goes only when neither leaves 2.
  const uint32_t vBytes = (uint32_t)q.N1 * 512u;
  const bool w200 = (p.D + 199) / 200 * 200 < (p.D + 127) / 128 * 128;
  const int widths[2] = {w200 ? 200 : 128, w200 ? 128 : 200};
  Geometry first{};
  for (int NW : widths) {
    Geometry t = q;
    t.N2 = NW;
    t.stage2Bytes = 2u * (uint32_t)NW * 128u;
    if (vBytes + 2u * t.stage2Bytes > ring) continue;
    t.nS1 = nS1;
    t.nS2 = (int)((ring - vBytes) / t.stage2Bytes); if (t.nS2 > kMaxS2) t.nS2 = kMaxS2;
    t.ok = true;
    if (!want_prefetch) return t;
    if (!first.ok) first = t;
    // both GEMMs give up stages (never below 2) until both prefetch warps have kMaxPf row slots
    const uint32_t want = 2u * kMaxPf * row;
    int s1 = t.nS1, s2 = t.nS2;
    while (s1 > 2 && ring - (uint32_t)s1 * fp1 < want) --s1;
    while (s2 > 2 && ring - (vBytes + (uint32_t)s2 * t.stage2Bytes) < want) --s2;
    uint32_t used = (uint32_t)s1 * fp1;
    if (vBytes + (uint32_t)s2 * t.stage2Bytes > used) used = vBytes + (uint32_t)s2 * t.stage2Bytes;
    int slots = (int)((ring - used) / (2u * row));
    if (slots > kMaxPf) slots = kMaxPf;
    if (slots >= 2) { t.pf_slots = slots; t.nS1 = s1; t.nS2 = s2; t.pf_off = used; return t; }
  }
  return first;
}

int launch_error() {
  const cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? KGE_OK : fail(KGE_ERR_CUDA, "k_fused launch: %s", cudaGetErrorString(e));
}
// k_fused<P>'s launch name carries the variant and the ring layout, so a profile says which one ran: GEMM1 width NV,
// GEMM2 chunk NW, prefetch slots per warp and the number of V hand-off warps
const char* pos_launch_name(int NV, int NW, int pf) {
  static const int nvs[4] = {64, 128, 208, 256}, nws[2] = {128, 200};
  static char names[4][2][kMaxPf + 1][96];
  static std::once_flag once;
  std::call_once(once, [] {
    for (int a = 0; a < 4; ++a)
      for (int b = 0; b < 2; ++b)
        for (int f = 0; f <= kMaxPf; ++f)
          snprintf(names[a][b][f], sizeof(names[a][b][f]), "k_fused<P: S=A.Bn^T, loss, GA=V.Bn> NV=%d NW=%d pf=%d hand=%d",
                   nvs[a], nws[b], f, f > 0 ? 1 : 3);
  });
  const int a = NV == 64 ? 0 : NV == 128 ? 1 : NV == 208 ? 2 : 3;
  return names[a][NW == 200][pf < 0 ? 0 : (pf > kMaxPf ? kMaxPf : pf)];
}
template <int NV, int NW>
int launch_pos(const LaunchCtx& c, int grid, size_t smem, const CUtensorMap* m, const FusedArgs& g) {
  if (int rc = smem_optin((const void*)k_fused_pos<NV, NW>, smem)) return rc;
  KGE_LAUNCH_NAMED(c, pos_launch_name(NV, NW, g.pf_slots), (k_fused_pos<NV, NW>), grid, kThreadsF, smem,
                   m[0], m[1], m[2], m[3], m[4], m[5], g);
  return launch_error();
}
template <int NV>
int launch_pos(const LaunchCtx& c, int grid, size_t smem, const CUtensorMap* m, const FusedArgs& g) {
  // geometry() never pairs N1 = 256 with NW = 200: the 128 KB V buffer and two 50 KB stages exceed the ring
  if constexpr (NV < 256) {
    if (g.N2 == 200) return launch_pos<NV, 200>(c, grid, smem, m, g);
  }
  return launch_pos<NV, 128>(c, grid, smem, m, g);
}
template <int NW, bool FLAT>
int launch_neg_src(const LaunchCtx& c, int grid, size_t smem, const CUtensorMap* m, const FusedArgs& g) {
  if (int rc = smem_optin((const void*)k_fused_neg<NW, FLAT>, smem)) return rc;
  // the launch name carries the output-column chunk width, so a profile says which variant ran
  static char name[64];
  static std::once_flag once;
  std::call_once(once, [] { snprintf(name, sizeof(name), "k_fused<N: G_neg=V^T.A, mean sq> NW=%d", NW); });
  KGE_LAUNCH_NAMED(c, name, (k_fused_neg<NW, FLAT>), grid, kThreadsF, smem, m[0], m[1], m[2], m[3], g);
  return launch_error();
}
template <int NW>
int launch_neg(const LaunchCtx& c, int grid, size_t smem, const CUtensorMap* m, const FusedArgs& g) {
  return (g.xraw || g.xids) ? launch_neg_src<NW, true>(c, grid, smem, m, g) : launch_neg_src<NW, false>(c, grid, smem, m, g);
}
int launch_width(const LaunchCtx& c, bool P, int grid, size_t smem, const CUtensorMap* m, const FusedArgs& g) {
  switch (g.N1) {
    case 64: return P ? launch_pos<64>(c, grid, smem, m, g) : launch_neg<64>(c, grid, smem, m, g);
    case 128: return P ? launch_pos<128>(c, grid, smem, m, g) : launch_neg<128>(c, grid, smem, m, g);
    case 200: return launch_neg<200>(c, grid, smem, m, g);
    case 208: return launch_pos<208>(c, grid, smem, m, g);
    default: return P ? launch_pos<256>(c, grid, smem, m, g) : launch_neg<256>(c, grid, smem, m, g);
  }
}
}  // namespace

int fused_prefetch_slots(const StepParams& p, int mode) { return geometry(p, mode, true).pf_slots; }

FusedHilo fused_hilo(const StepParams& p) {
  // k_fused<P>'s GEMM1 width does not depend on prefetch; k_fused<N> is 256 wide only without it
  return FusedHilo{!k_reg_a(geometry(p, 0, false).N1), !k_reg_a(neg_chunk_width(p.D, false))};
}

int fused_launch(const LaunchCtx& c, const StepParams& p, const StepWs& w, int mode, const float* wt, float* dumpS,
                 float* dumpV, const TableView* ent, const long long* neg_ids, const FusedPrefetch* pf) {
  FusedArgs g{};
  g.model = p.model; g.adversarial = p.adversarial;
  g.gamma = p.gamma; g.Tl2e = p.adv_temperature * kLog2e; g.inv2B = 0.5f / (float)p.B; g.uni = 1.f / (float)p.Ns;
  g.reg_coef = p.reg_coef; g.reg_norm = p.reg_norm;
  g.C = p.C; g.D = p.D; g.nblkD = slab_blocks(p.D);
  const bool P = mode == 0;
  const Geometry q = geometry(p, mode, pf != nullptr && ent != nullptr);
  if (!q.ok) return fail(KGE_ERR_UNSUPPORTED, "fused kernel: shape does not fit (N1=%d)", q.N1);
  g.Rx = q.Rx; g.Ry = q.Ry; g.N1 = q.N1; g.N2 = q.N2; g.nS1 = q.nS1; g.nS2 = q.nS2;
  g.stage1Bytes = q.stage1Bytes; g.stage2Bytes = q.stage2Bytes;
  if (pf && ent && q.pf_slots >= 2) {
    static const int lag_env = getenv("KGE_B200_PF_LAG") ? atoi(getenv("KGE_B200_PF_LAG")) : 1;
    g.pf_lag = lag_env < 1 ? 1 : (lag_env > 3 ? 3 : lag_env);
    g.pf_slots = q.pf_slots; g.pf_off = q.pf_off; g.pf_row_bytes = (uint32_t)p.D * 4u; g.pf_parity = mode;
    g.pf_node_ids = pf->node_ids; g.pf_nU_dev = pf->nU_dev; g.pf_nU = pf->nU; g.pf_nNeg = pf->nNeg;
    g.pf_neg_ids = pf->neg_ids; g.pf_nc = pf->nc; g.pf_bn = pf->bn;
    g.xtab = *ent;
  }
  // the coefficients go over as fp32, or as hi/lo when k_fused<N> runs 256 columns wide (both launches see the same
  // prefetch decision, so P writes what N reads)
  if (k_reg_a(geometry(p, 1, pf != nullptr && ent != nullptr).N1)) g.VT = w.VT;
  else { g.VhiT = w.VhiT; g.VloT = w.VloT; }
  g.colpart = w.colpart; g.ncolpart = (p.Cs + kTileM - 1) / kTileM;
  g.dumpV = dumpV;
  const size_t smem = q.ringBytes + 1024;
  const int mtiles = (g.Rx + kTileM - 1) / kTileM;
  int grid = p.C * mtiles;
  if (grid > c.num_sms) grid = c.num_sms;
  CUtensorMap m[6];
  if (P) {
    g.x2 = w.a2; g.y2 = w.b2;
    g.pos = w.pos; g.wt = wt; g.wbar = w.wbar;
    g.gpos = w.gpos; g.rowsum = w.rowsum; g.pl = w.pl; g.nl = w.nl;
    g.dumpS = dumpS;
    g.out = w.GA;
    // GEMM2 contracts over the negatives: its operand is the transposed slab copy of Bn
    const long long rowsX = (long long)p.C * p.Cs * g.nblkD, rowsY = (long long)p.C * p.Ns * g.nblkD;
    const long long rowsYT = (long long)p.C * slab_blocks(p.Ns) * p.D;
    const bool ra = k_reg_a(g.N1);
    if (tc_make_map(&m[0], ra ? w.Af : w.Ahi, rowsX, 32, kTileM) || tc_make_map(&m[1], ra ? w.Af : w.Alo, rowsX, 32, kTileM) ||
        tc_make_map(&m[2], w.Bhi, rowsY, 32, g.N1) || tc_make_map(&m[3], w.Blo, rowsY, 32, g.N1) ||
        tc_make_map(&m[4], w.BhiT, rowsYT, 32, g.N2) || tc_make_map(&m[5], w.BloT, rowsYT, 32, g.N2))
      return KGE_ERR_CUDA;
    return launch_width(c, true, grid, smem, m, g);
  }
  g.Xhi = w.Bhi; g.Xlo = w.Blo;
  // one GPU: the negatives' own rows come straight from the table (exact fp32, one load); sharded tables would make
  // that a remote read per row, so they use the local hi + lo slabs
  if (ent && ent->n_shards == 1 && neg_ids) { g.xids = neg_ids; g.xtab = *ent; }
  if (w.BnRaw) g.xraw = w.BnRaw;
  g.gsn = w.gsn;
  g.out = w.Bn;
  // A operand: the fp32 V^T slab [C][Cs/32][Ns][32]; B operand: A^T slabs [C][Cs/32][D][32]; K = i
  const long long rowsV = (long long)p.C * slab_blocks(p.Cs) * p.Ns, rowsA = (long long)p.C * slab_blocks(p.Cs) * p.D;
  const bool rv = k_reg_a(g.N1);
  if (tc_make_map(&m[0], rv ? w.VT : w.VhiT, rowsV, 32, kTileM) || tc_make_map(&m[1], rv ? w.VT : w.VloT, rowsV, 32, kTileM) ||
      tc_make_map(&m[2], w.AhiT, rowsA, 32, g.N1) || tc_make_map(&m[3], w.AloT, rowsA, 32, g.N1))
    return KGE_ERR_CUDA;
  return launch_width(c, false, grid, smem, m, g);
}

}  // namespace kge
