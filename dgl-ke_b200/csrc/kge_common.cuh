// kge_common.cuh -- shared device helpers for libkge_b200 (sm_90a).
//
// Data model (DESIGN.md "HBM layout"):
//   * embedding tables: fp32 row-major, row-range sharded over <= 8 GPUs (TableView); a row
//     address on a remote shard is a peer-mapped pointer, so every kernel below works unchanged
//     over NVLink (loads for the gather, red.add for the Adagrad scatter).
//   * per-step workspace (StepWs): dense fp32 matrices that stay L2-resident between phases.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "../../include/kge_b200.h"

namespace kge {

constexpr int kWarp = 32;

struct TableView {
  float* emb[KGE_MAX_SHARDS];
  float* state[KGE_MAX_SHARDS];
  long long rows_per_shard;
  long long num_rows;
  int n_shards;
  int dim;
};

__device__ __forceinline__ float* row_ptr(const TableView& t, long long id) {
  if (t.n_shards == 1) return t.emb[0] + id * (long long)t.dim;
  int s = (int)(id / t.rows_per_shard);
  return t.emb[s] + (id - (long long)s * t.rows_per_shard) * (long long)t.dim;
}
__device__ __forceinline__ float* state_ptr(const TableView& t, long long id) {
  if (t.n_shards == 1) return t.state[0] + id;
  int s = (int)(id / t.rows_per_shard);
  return t.state[s] + (id - (long long)s * t.rows_per_shard);
}

// Scalars of one step, passed by value to every kernel.
struct StepParams {
  int model;
  int D;        // entity row length
  int Dr;       // relation row length
  float gamma, emb_init, lr, reg_coef;
  int reg_norm;
  int adversarial;
  float adv_temperature;
  int neg_head;
  long long B;  // positives
  int C, Cs, Ns;
  long long Nn; // C * Ns negative rows
  long long U;  // unique positive nodes (capacity 2B when only the device knows the count: U_dev)
  const long long* U_dev;   // device-side node count (device sampler) or null
  int rel_deferred;  // 1: relation Adagrad is applied later from dense all-reduced buffers (multi-GPU)
  int rel_dense;     // 1: k_chain sums relation gradients per relation into ws.rg / ws.rgs (fused single-GPU step)
  int use_nc;        // 1: head/tail rows are read from the gathered copy NC (3-call API, sharded tables); 0: from the table
  int fused;         // 1: contraction by the fused wgmma kernel (kge_fused.cu): operands exist only as slabs
  int hinge;         // 1: Hinge criterion (loss.py:10-17); 0: Logsigmoid == Logistic == BCE
  float margin;      // Hinge margin
  int pairwise;      // 1: criterion(pos_i - neg_ij, +1), plain mean over all (i, j) (loss.py:76-80)
  int neg_deg;       // 1: --neg_deg_sample: Ns = chunk_size + sampled negatives, the first Cs rows of a chunk's negatives are
                     //    the chunk's own corrupted-side rows (kge_negdeg.cu)
  int nc_staged;     // 1: NC was filled by the previous step's prefetch warps (kge_set_next_batch): no k_gather_nodes ran
};

// who produces the unique nodes' share of the regulariser: k_gather_nodes when it runs, else the node update
__host__ __device__ __forceinline__ bool node_reg_in_update(const StepParams& p) { return !p.use_nc || p.nc_staged; }

// Device workspace of one step (all pointers into the handle's arena).
struct StepWs {
  float* A;        // [B, D]   a-side rows (h+r, t-r, h*r, ...)
  float* Bn;       // [Nn, D]  gathered negative rows; overwritten by their gradient
  float* GA;       // [B, D]   d loss / d a
  float* GR;       // [B, Dr]  d loss / d relation rows (per edge)
  float* NG;       // [U, D]   d loss / d unique positive nodes (without reg), zero between steps
  float* NC;       // [U, D]   gathered rows of the unique positive nodes (= pos_g.ndata['emb'], general_models.py:548):
                   //          every later read of a head/tail row is local, even when the table is sharded over GPUs
  float* S;        // [B, Ns]  negative scores
  float* V;        // [B, Ns]  backward coefficients
  float* pos;      // [B]
  float* gpos;     // [B]      d loss / d pos
  float* pnorm;    // [B]      |h+r-t| (TransE_l2)
  float* a2;       // [B]      |a|^2 (TransE_l2)
  float* b2;       // [Nn]     |b|^2 (TransE_l2)
  float* rowsum;   // [B]      sum_j V_ij (TransE_l2)
  float* colsum;   // [Nn]     sum_i V_ij (TransE_l2)
  float* pl;       // [B]      positive loss terms
  float* nl;       // [B]      negative loss terms (already reduced over j)
  float* regp;     // [B + Nn + U] partial sums of |x|^p
  float* wbar;     // [1]      mean edge weight
  float* gsr;      // [B]      mean(GR_i^2) per edge (relation Adagrad phase 1)
  float* gsn;      // [Nn]     mean(G_neg_j^2) per negative row (fused kernel, mode N)
  float* colpart;  // [ceil(Cs/128)][Nn] sum_i V_ij over each 128-row tile of positives (fused kernel: mode P -> mode N)
  float* rg;       // [n_rel, Dr] dense per-relation gradient sums (rel_dense), zero between steps
  float* rgs;      // [n_rel]     dense per-relation sums of mean(g^2)          , zero between steps
  const float* BnRaw;         // [Nn, D] negative rows staged by the previous step's prefetch warps, or null
  unsigned int* sync_ctr;     // [4] grid-barrier counters of k_update (zero between launches)
  float* red_partial;         // [64 * 3] partial sums of k_reduce_log
  unsigned int* red_ticket;   // [1] completion ticket of k_reduce_log (zero between launches)
  float* Mt;       // [B, D]   RESCAL: M_r t  (tail mode needs it next to A = M_r h)
  // wgmma engine: TF32 hi/lo splits of the contraction operands
  float *Ahi, *Alo;   // [C][D/32][Cs][32]   (slab layout, see slab_off)
  float *Bhi, *Blo;   // [C][D/32][Ns][32]
  float *Vhi, *Vlo;   // [C][Ns/32][Cs][32]
  // the same operands transposed (see slabT_off): wgmma takes TF32 operands K-major only, and the gradient GEMMs
  // contract over the rows of these matrices
  float *AhiT, *AloT; // [C][Cs/32][D][32]
  float *BhiT, *BloT; // [C][Ns/32][D][32]
  float *VhiT, *VloT; // [C][Cs/32][Ns][32]   (stand-alone engine)
  // fused step: the operands that are only ever the A operand of a fused GEMM, stored once as fp32 and split into TF32
  // hi/lo in registers by the warp that issues the wgmma (kge_fused.cu); these replace Ahi/Alo and VhiT/VloT there,
  // except next to a 256-wide accumulator (fused_hilo)
  float* Af;          // [C][D/32][Cs][32]   (slab layout, written by k_prep, the A operand of GEMM1 in mode P)
  float* VT;          // [C][Cs/32][Ns][32]   (written by mode P, the A operand of mode N)
};

struct BatchView {
  const long long* node_ids;
  const long long* head_local;
  const long long* tail_local;
  const long long* rel_ids;
  const long long* neg_ids;
  const float* edge_weight;
  const long long* head_ids;    // optional global ids of the edges' endpoints
  const long long* tail_ids;
};

__device__ __forceinline__ long long node_count(const StepParams& p) { return p.U_dev ? *p.U_dev : p.U; }

// row of the positive graph's local node `loc` (pos_g.ndata['emb'][loc], general_models.py:548): the gathered copy,
// or the table row itself when nothing can have changed it since the gather (single-GPU fused step)
__device__ __forceinline__ const float* node_row(const StepParams& p, const TableView& ent, const BatchView& b,
                                                 const StepWs& w, long long loc) {
  return p.use_nc ? (w.NC + loc * (long long)p.D) : row_ptr(ent, b.node_ids[loc]);
}
// head / tail row of edge i: with the edges' global ids at hand the table row needs one index load instead of two
__device__ __forceinline__ const float* head_row(const StepParams& p, const TableView& ent, const BatchView& b,
                                                 const StepWs& w, long long i) {
  if (!p.use_nc && b.head_ids) return row_ptr(ent, b.head_ids[i]);
  return node_row(p, ent, b, w, b.head_local[i]);
}
__device__ __forceinline__ const float* tail_row(const StepParams& p, const TableView& ent, const BatchView& b,
                                                 const StepWs& w, long long i) {
  if (!p.use_nc && b.tail_ids) return row_ptr(ent, b.tail_ids[i]);
  return node_row(p, ent, b, w, b.tail_local[i]);
}

// ------------------------------------------------------------------------------------------
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

__device__ __forceinline__ float4 ld4(const float* p) { return *reinterpret_cast<const float4*>(p); }
__device__ __forceinline__ void st4(float* p, float4 v) { *reinterpret_cast<float4*>(p) = v; }
// streaming (read-once) table row load: do not allocate in L1
__device__ __forceinline__ float4 ld4_stream(const float* p) {
  float4 r;
  asm volatile("ld.global.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
  return r;
}
// vector fp32 reduction into global / peer memory (sm_90+: one 16-byte RED instead of four)
__device__ __forceinline__ void red_add4(float* p, float4 v) {
  asm volatile("red.global.add.v4.f32 [%0], {%1,%2,%3,%4};"
               :: "l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}

// system-scope variants for rows that may live in a peer GPU's HBM (NVLink atomics)
__device__ __forceinline__ void red_add4_sys(float* p, float4 v) {
  asm volatile("red.relaxed.sys.global.add.v4.f32 [%0], {%1,%2,%3,%4};"
               :: "l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
__device__ __forceinline__ void table_red_add4(const TableView& t, float* p, float4 v) {
  if (t.n_shards > 1) red_add4_sys(p, v); else red_add4(p, v);
}
__device__ __forceinline__ void table_atomic_add(const TableView& t, float* p, float v) {
  if (t.n_shards > 1) atomicAdd_system(p, v); else atomicAdd(p, v);
}

#define KGE_F4_OP2(name, expr)                                                     \
  __device__ __forceinline__ float4 name(float4 a, float4 b) {                     \
    float4 r;                                                                      \
    { float x = a.x, y = b.x; r.x = (expr); } { float x = a.y, y = b.y; r.y = (expr); } \
    { float x = a.z, y = b.z; r.z = (expr); } { float x = a.w, y = b.w; r.w = (expr); } \
    return r;                                                                      \
  }
KGE_F4_OP2(f4_add, x + y)
KGE_F4_OP2(f4_sub, x - y)
KGE_F4_OP2(f4_mul, x* y)
#undef KGE_F4_OP2
__device__ __forceinline__ float4 f4_scale(float4 a, float s) { return make_float4(a.x * s, a.y * s, a.z * s, a.w * s); }
__device__ __forceinline__ float4 f4_neg(float4 a) { return make_float4(-a.x, -a.y, -a.z, -a.w); }
__device__ __forceinline__ float4 f4_fma(float4 a, float s, float4 c) {
  return make_float4(fmaf(a.x, s, c.x), fmaf(a.y, s, c.y), fmaf(a.z, s, c.z), fmaf(a.w, s, c.w));
}
__device__ __forceinline__ float f4_hsum(float4 a) { return (a.x + a.y) + (a.z + a.w); }
__device__ __forceinline__ float f4_dot(float4 a, float4 b) { return f4_hsum(f4_mul(a, b)); }
__device__ __forceinline__ float sgnf(float x) { return (x > 0.f) ? 1.f : ((x < 0.f) ? -1.f : 0.f); }

// 3xTF32 operand split: x = hi + lo with hi = rna_tf32(x), lo = rna_tf32(x - hi)
__device__ __forceinline__ void split_tf32(float x, float& hi, float& lo) {
  uint32_t hb, lb;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(hb) : "f"(x));
  hi = __uint_as_float(hb);
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(lb) : "f"(x - hi));
  lo = __uint_as_float(lb);
}
__device__ __forceinline__ void split_tf32_4(float4 v, float4& h, float4& l) {
  split_tf32(v.x, h.x, l.x); split_tf32(v.y, h.y, l.y); split_tf32(v.z, h.z, l.z); split_tf32(v.w, h.w, l.w);
}
// wgmma operand layout ("k-blocked slabs"): a per-chunk matrix X[c][row][col] (row < R, col < Ncol) is stored as
//   X[c][col / 32][row][col % 32]
// so that every TMA box the GEMMs load -- {32 cols, n rows} of one (chunk, 32-column block) -- is ONE contiguous
// n*128-byte region of HBM (the row-major layout made each box 128..208 scattered 128-byte lines).
__host__ __device__ inline int slab_blocks(int ncol) { return (ncol + 31) >> 5; }
__device__ __forceinline__ long long slab_off(long long chunk, int nblk, int R, int row, int col) {
  return ((chunk * nblk + (col >> 5)) * (long long)R + row) * 32 + (col & 31);
}
// transposed slabs: the same matrix stored as X^T[c][row / 32][col][row % 32] (Ncol rows of 32 consecutive `row`s), the
// K-major form of X when the contraction runs over its rows
__device__ __forceinline__ long long slabT_off(long long chunk, int R, int Ncol, int row, int col) {
  return ((chunk * slab_blocks(R) + (row >> 5)) * (long long)Ncol + col) * 32 + (row & 31);
}
// k_prep stages 32 operand rows in shared memory to write their transposed slabs as whole lines (kge_rows.cu).  Row
// stride (floats): >= D and = 4 (mod 32), so that both the float4 stores along a row (8 lanes = 128 contiguous bytes) and
// the float4 loads of one column group by 8 consecutive rows (8 distinct 16-byte bank groups) are free of bank conflicts.
constexpr int kPrepRows = 32;                         // = the row extent of one transposed slab block
constexpr size_t kSmemOptinMax = 227 * 1024;          // per-block opt-in shared memory of sm_90
__host__ __device__ inline int prep_stage_stride(int D) { return ((D + 27) & ~31) + 4; }
inline size_t prep_stage_bytes(int D) { return (size_t)kPrepRows * prep_stage_stride(D) * sizeof(float); }
// the wgmma engine (transposed slabs) is offered only where k_prep's staging buffer fits one CTA: D <= 1796
inline bool prep_stage_fits(int D) { return prep_stage_bytes(D) <= kSmemOptinMax; }

// destination of an operand row: plain fp32 row-major and/or its TF32 hi/lo split in slab layout and/or fp32 in slab
// layout, and/or a copy in shared memory (k_prep writes the transposed slabs from there)
struct RowOut {
  float* f32;        // row-major row pointer or null
  float* hi;         // slab-layout base pointers or null
  float* lo;
  long long chunk;
  int nblk, R, row;
  float* stage;      // shared-memory row or null
  float* slab;       // slab-layout base pointer of the unsplit fp32 row or null
};
__device__ __forceinline__ void row_store4(const RowOut& o, int col, float4 v) {
  if (o.f32) *reinterpret_cast<float4*>(o.f32 + col) = v;
  if (o.hi || o.slab) {
    const long long off = slab_off(o.chunk, o.nblk, o.R, o.row, col);
    if (o.slab) *reinterpret_cast<float4*>(o.slab + off) = v;
    if (o.hi) {
      float4 h, l;
      split_tf32_4(v, h, l);
      *reinterpret_cast<float4*>(o.hi + off) = h;
      *reinterpret_cast<float4*>(o.lo + off) = l;
    }
  }
  if (o.stage) *reinterpret_cast<float4*>(o.stage + col) = v;
}

// |x|^p  and  d/dx coef*|x|^p  (general_models.py:572-576: coef * norm(x, p)**p)
static __device__ __noinline__ float abs_pow_generic(float ax, int p) { return powf(ax, (float)p); }
__device__ __forceinline__ float abs_pow(float x, int p) {
  float ax = fabsf(x);
  if (p == 3) return ax * ax * ax;
  if (p == 2) return ax * ax;
  if (p == 1) return ax;
  return abs_pow_generic(ax, p);
}
// the powf path is kept out of line: inlined at every call site it multiplied the code size of the kernels that apply
// the regulariser per element (the fused kernel's negative-side pass went from 4k to 12k instructions and thrashed the
// instruction cache), and no reference recipe uses a norm other than 1, 2 or 3
static __device__ __noinline__ float reg_grad_pow(float x, int p, float coef) {
  return coef * (float)p * powf(fabsf(x), (float)(p - 1)) * sgnf(x);
}
__device__ __forceinline__ float reg_grad(float x, int p, float coef) {
  if (coef == 0.f || p <= 0) return 0.f;
  float ax = fabsf(x);
  if (p == 3) return 3.f * coef * ax * x;
  if (p == 2) return 2.f * coef * x;
  if (p == 1) return coef * sgnf(x);
  return reg_grad_pow(x, p, coef);
}
__device__ __forceinline__ float4 reg_grad4(float4 x, int p, float coef) {
  return make_float4(reg_grad(x.x, p, coef), reg_grad(x.y, p, coef), reg_grad(x.z, p, coef), reg_grad(x.w, p, coef));
}
__device__ __forceinline__ float abs_pow4_sum(float4 x, int p) {
  return (abs_pow(x.x, p) + abs_pow(x.y, p)) + (abs_pow(x.z, p) + abs_pow(x.w, p));
}

// -logsigmoid(-s) = softplus(s);  sigmoid(s)
__device__ __forceinline__ float softplusf(float s) { return fmaxf(s, 0.f) + log1pf(expf(-fabsf(s))); }
__device__ __forceinline__ float sigmoidf(float s) {
  // stable on both tails
  if (s >= 0.f) return 1.f / (1.f + expf(-s));
  float e = expf(s);
  return e / (1.f + e);
}

inline int ceil_div(long long a, long long b) { return (int)((a + b - 1) / b); }

// ------------------------------------------------------------------------------------------
// host-side launchers and engines
//
// Errors: every host function that returns an int returns a KGE_* code and, when it is not KGE_OK, has already set the
// message kge_last_error() returns (fail(), kge_abi.cu).  The void launchers only enqueue a kernel; their launch errors
// are picked up by the caller's cudaGetLastError.
int fail(int code, const char* fmt, ...);
// Opts `kernel` in to `bytes` of dynamic shared memory on the current device when that exceeds the 48 KB default.  The
// attribute belongs to the (kernel, device) pair; the largest size set so far is remembered, so only a larger size
// costs a driver call.
int smem_optin(const void* kernel, size_t bytes);

// Optional per-launch timing (kge_profile_*): CUDA events recorded on the launching stream
// around every kernel of a step; read back after a stream sync.
struct Profiler {
  static constexpr int kMax = 64;
  bool enabled = false;
  int n = 0;
  const char* names[kMax];
  cudaEvent_t ev0[kMax], ev1[kMax];
  bool created = false;
};

struct LaunchCtx {
  cudaStream_t stream;
  long long* launch_counter;
  int num_sms;
  Profiler* prof;
};

inline void prof_begin(const LaunchCtx& c, const char* name) {
  Profiler* p = c.prof;
  if (!p || !p->enabled || p->n >= Profiler::kMax) return;
  p->names[p->n] = name;
  cudaEventRecord(p->ev0[p->n], c.stream);
}
inline void prof_end(const LaunchCtx& c) {
  Profiler* p = c.prof;
  if (!p || !p->enabled || p->n >= Profiler::kMax) return;
  cudaEventRecord(p->ev1[p->n], c.stream);
  ++p->n;
}

#define KGE_LAUNCH_NAMED(ctx, name, kernel, grid, block, smem, ...)            \
  do {                                                                          \
    prof_begin((ctx), name);                                                    \
    kernel<<<(grid), (block), (smem), (ctx).stream>>>(__VA_ARGS__);             \
    prof_end((ctx));                                                            \
    if ((ctx).launch_counter) ++*(ctx).launch_counter;                          \
  } while (0)

#define KGE_LAUNCH(ctx, kernel, grid, block, smem, ...)                         \
  do {                                                                          \
    prof_begin((ctx), #kernel);                                                 \
    kernel<<<(grid), (block), (smem), (ctx).stream>>>(__VA_ARGS__);             \
    prof_end((ctx));                                                            \
    if ((ctx).launch_counter) ++*(ctx).launch_counter;                          \
  } while (0)

// device-side sampler (kge_sampler.cu)
struct SamplerParams {
  const long long *heads, *rels, *tails;   // the partition's edges (device)
  long long n_edges, n_entities;
  long long B, Nn;
  unsigned long long seed;
  int half_bits;                            // Feistel half width: 2^(2*half_bits) >= n_edges
  // outputs
  long long *o_head, *o_rel, *o_tail;       // [B] global ids of the sampled positives
  long long *o_neg;                         // [Nn]
  long long *o_nodes, *o_hl, *o_tl;         // [2B], [B], [B]
  long long* o_n_nodes;                     // [1]
  // hash table of the batch's distinct entity ids
  unsigned long long* tkey;                 // [H], ~0 = empty
  int* tpos;                                // [H] smallest position of the key in [heads | tails]
  int* tloc;                                // [H] local id of the key
  int hmask;                                // H - 1
  int* flags;                               // [2B] 1 = first occurrence
};

void launch_sampler(const LaunchCtx&, const SamplerParams&, long long step);

// row kernels (kge_rows.cu, kge_tiles.cu)
void launch_gather(const LaunchCtx&, const TableView& t, const long long* idx, long long n, float* out);
void launch_gather_nodes(const LaunchCtx&, const StepParams&, const TableView& ent, const BatchView&, const StepWs&);
int launch_prep(const LaunchCtx&, const StepParams&, const TableView& ent, const TableView& rel,
                const BatchView&, const StepWs&);
// k_prep's negative-row blocks only (RESCAL computes its edge rows in its own kernel)
int launch_prep_nonedge(const LaunchCtx&, const StepParams&, const TableView& ent, const TableView& rel,
                        const BatchView&, const StepWs&);
// dense-row variant used by kge_score_pos / kge_score_neg (rows already gathered)
void launch_prep_dense(const LaunchCtx&, const StepParams&, const float* head, const float* relr,
                       const float* tail, const float* negrows, const StepWs&, bool want_pos, bool want_a);
void launch_score(const LaunchCtx&, const StepParams&, const StepWs&);
void launch_loss(const LaunchCtx&, const StepParams&, const float* pos, const float* S, const float* w,
                 const StepWs&, float* log4, bool want_reg);
void launch_wbar(const LaunchCtx&, const StepParams&, const float* w, const StepWs&);
void launch_loss_rows(const LaunchCtx&, const StepParams&, const float* pos, const float* S, const float* w, const StepWs&);
void launch_colsum(const LaunchCtx&, const StepParams&, const StepWs&);
void launch_reduce_log(const LaunchCtx&, const StepParams&, const float* w, const StepWs&, float* log4, bool want_reg);
void launch_grad_a(const LaunchCtx&, const StepParams&, const StepWs&);
void launch_grad_b(const LaunchCtx&, const StepParams&, const StepWs&);
void launch_chain(const LaunchCtx&, const StepParams&, const TableView& ent, const TableView& rel,
                  const BatchView&, const StepWs&);
// ExternalEmbedding.update of the step's three trace entries; log4 != null also reduces the log scalars (fused step)
int launch_update(const LaunchCtx&, const StepParams&, const TableView& ent, const TableView& rel,
                  const BatchView&, const StepWs&, float* log4, const float* wt);
void launch_adagrad(const LaunchCtx&, const TableView& t, const long long* idx, const float* grad,
                    long long n, float lr);
void launch_node_grad_with_reg(const LaunchCtx&, const StepParams&, const TableView& ent,
                               const BatchView&, const StepWs&, float* out);
void launch_fill_zero(const LaunchCtx&, float* p, long long n);
void launch_rel_grad_dense(const LaunchCtx&, const StepParams&, const BatchView&, const StepWs&, float* rg, float* rgs);
void launch_rel_apply_dense(const LaunchCtx&, const TableView& rel, float* rg, float* rgs, float lr);

// --neg_deg_sample fix-up kernels (kge_negdeg.cu)
void launch_negdeg_ids(const LaunchCtx&, const StepParams&, const BatchView&, const long long* sampled, long long* out);
void launch_negdeg_zero_reg(const LaunchCtx&, const StepParams&, const StepWs&);
void launch_negdeg_mask_scores(const LaunchCtx&, const StepParams&, const StepWs&);
void launch_negdeg_mask_coef(const LaunchCtx&, const StepParams&, const StepWs&);
void launch_negdeg_scatter(const LaunchCtx&, const StepParams&, const TableView& ent, const BatchView&, const StepWs&);

// filtered ranking of evaluation queries over one score tile (kge_eval.cu)
struct RankParams {
  const float* S;               // [Q, ld] score tile, N columns used
  long long ld, Q, N;
  const float* pos;             // [Q]
  long long base;               // range ids: column j is entity base + j (cand == null)
  const long long* cand;        // explicit ids: [Q / chunk, N], query q reads row q / chunk
  long long chunk;
  const long long* kept;        // [Q] the query's kept-side entity and its relation: key = kept * n_rel + rel
  const long long* rel;
  const long long* keys;        // [n_keys] sorted, or null: no filter
  const int* vals;              // [n_keys] sorted and distinct within each key
  long long n_keys, n_rel;
  long long* cnt;               // [Q]
};
void launch_rank_count(const LaunchCtx&, const RankParams&);
void launch_rank_finish(const LaunchCtx&, const long long* cnt, long long Q, long long* rank_out, double* acc);

// running top-K lists over one score tile (kge_topk.cu)
constexpr int kTopkSeg = 4096;            // columns per select CTA
struct TopkParams {
  const float* S;               // [Q, ld] score tile, N columns used
  long long ld, Q, N;
  const long long* qgroup;      // [Q] list of each row (a list's rows are consecutive)
  const long long* qoff;        // [Q] key of (q, j) = qoff[q] + (cbase + j) * cstride
  long long cbase, cstride;
  int K;
  float* top_score;             // [G, K] in list order, empty slots -inf / -1
  long long* top_key;
  // workspace (topk_carve): the select CTAs' survivors [Q * nseg, K], their counts, the per-list bound [G]
  float* cs;
  long long* ck;
  int* cn;
  unsigned* bound;
};
size_t topk_workspace_bytes(long long Q, long long N, int K, long long G);
void topk_carve(TopkParams& p, void* ws);
void launch_topk(const LaunchCtx&, const TopkParams&);

// embedding similarity tiles (kge_sim.cu)
bool sim_uses_gemm(int sim);
size_t sim_workspace_bytes(long long nL, long long nR, int dim);       // the GEMM functions' TF32 operands and norms
int launch_sim_tile(const LaunchCtx&, int sim, const float* L, long long nL, const float* R, long long nR, int dim,
                    float* S, void* ws);
void launch_sim_pairs(const LaunchCtx&, int sim, const float* L, const float* R, long long n, int dim, float* out);

// RESCAL-specific row kernels (kge_rescal.cu)
int launch_rescal_prep(const LaunchCtx&, const StepParams&, const TableView& ent, const TableView& rel,
                       const BatchView&, const StepWs&);
void launch_rescal_prep_dense(const LaunchCtx&, const StepParams&, const float* head, const float* relr,
                              const float* tail, const StepWs&, bool want_pos, bool want_a);
void launch_rescal_chain(const LaunchCtx&, const StepParams&, const TableView& ent, const TableView& rel,
                         const BatchView&, const StepWs&);

// wgmma engine (kge_umma.cu): the three contractions as stand-alone GEMMs, for the shapes umma_supported accepts
bool umma_supported(const StepParams&);
int umma_score(const LaunchCtx&, const StepParams&, const StepWs&);
int umma_grad(const LaunchCtx&, const StepParams&, const StepWs&, bool side_b);

// fused contraction (kge_fused.cu): mode 0 = P (scores, loss, GA), mode 1 = N (G_neg, mean squares)
// Rows of the NEXT step that the fused kernel's spare warps copy while it computes (kge_set_next_batch)
struct FusedPrefetch {
  const long long* node_ids;   // next batch's unique nodes
  const long long* nU_dev;     // their count on the device, or null
  long long nU;                // their count (capacity when nU_dev is set)
  const long long* neg_ids;
  long long nNeg;
  float* nc;                   // [nU, D] destination of the node rows
  float* bn;                   // [nNeg, D] destination of the negative rows
};
bool fused_supported(const StepParams&);
// row slots per prefetch warp the shape leaves room for (< 2: none)
int fused_prefetch_slots(const StepParams& p, int mode);
// A operands of the fused kernels that travel as TF32 hi/lo slabs instead of fp32 (their 256-wide variants): the
// a-side (Ahi/Alo instead of Af) and the coefficients (VhiT/VloT as well as VT: without prefetch slots only)
struct FusedHilo { bool a, v; };
FusedHilo fused_hilo(const StepParams& p);
int fused_launch(const LaunchCtx&, const StepParams&, const StepWs&, int mode, const float* wt, float* dumpS, float* dumpV,
                 const TableView* ent, const long long* neg_ids, const FusedPrefetch* pf);

}  // namespace kge
