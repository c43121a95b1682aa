// kge_negdeg.cu -- --neg_deg_sample (models/general_models.py:396-403, 417-424, 429-432).
//
// With the flag the reference puts the chunk's OWN corrupted-side rows (the heads of its positives when heads are being
// corrupted, else the tails) in front of the sampled negatives of every chunk (Ns' = chunk_size + neg_sample_size columns),
// multiplies the score of a positive against its own row by 0, and lets the gradient of those extra columns flow into the
// positive-node leaf -- they are not a traced tensor of their own: no regulariser term, no Adagrad entry.
//
// Here the step runs UNCHANGED over an augmented negative id list (every existing kernel sees Ns' ordinary negatives per
// chunk) and five small kernels put the differences right:
//   k_negdeg_ids          ids'[c, j] = id of the chunk's j-th own row (j < Cs) | sampled id (j >= Cs)
//   k_negdeg_zero_reg     the prepended rows' share of the regulariser log is 0
//   k_negdeg_mask_scores  S[c, i, i] = 0                     (between the score kernel and k_loss: value 0 in the loss / softmax)
//   k_negdeg_mask_coef    V[c, i, i] = 0 and its TF32 hi/lo copies   (after k_loss: no gradient)
//   k_negdeg_scatter      G'[c, j] - reg'(row) is added to the positive node's gradient NG, then G'[c, j] = 0, so that the
//                         update kernel's negative phases (state add, row scatter) see a zero gradient for those rows
// Single-GPU tables only; the contraction takes the stand-alone GEMM / tile kernels (Ns' exceeds the fused kernel's register budget
// at the usual shapes, and its epilogue has no mask).
#include "kge_common.cuh"

namespace kge {

namespace {
constexpr int kBlock = 256;

__global__ void __launch_bounds__(kBlock) k_negdeg_ids(StepParams p, BatchView b, const long long* __restrict__ sampled,
                                                       long long* __restrict__ out) {
  const long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= p.Nn) return;
  const long long c = k / p.Ns;
  const int j = (int)(k % p.Ns);
  if (j < p.Cs) {
    const long long e = c * p.Cs + j;
    out[k] = b.node_ids[p.neg_head ? b.head_local[e] : b.tail_local[e]];
  } else {
    out[k] = sampled[c * (long long)(p.Ns - p.Cs) + (j - p.Cs)];
  }
}

__global__ void __launch_bounds__(kBlock) k_negdeg_zero_reg(StepParams p, StepWs w) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;     // one per prepended row: (c, j < Cs)
  if (t >= p.B) return;
  const long long c = t / p.Cs;
  const int j = (int)(t % p.Cs);
  w.regp[p.B + c * p.Ns + j] = 0.f;
}

__global__ void __launch_bounds__(kBlock) k_negdeg_mask_scores(StepParams p, StepWs w) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;     // positive i, column i % Cs
  if (i >= p.B) return;
  const long long o = i * (long long)p.Ns + (i % p.Cs);
  w.S[o] = 0.f;
  // TransE_l2: V holds |a - b| at this point and k_loss divides the coefficient by it; an infinite distance makes the
  // masked coefficient (and its share of rowsum_i) exactly 0
  if (p.model == KGE_TRANSE_L2) w.V[o] = INFINITY;
}

__global__ void __launch_bounds__(kBlock) k_negdeg_mask_coef(StepParams p, StepWs w) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= p.B) return;
  const int il = (int)(i % p.Cs);
  const long long o = i * (long long)p.Ns + il;
  w.V[o] = 0.f;
  if (w.Vhi) {
    const long long so = slab_off(i / p.Cs, slab_blocks(p.Ns), p.Cs, il, il);
    w.Vhi[so] = 0.f;
    w.Vlo[so] = 0.f;
    const long long st = slabT_off(i / p.Cs, p.Cs, p.Ns, il, il);
    w.VhiT[st] = 0.f;
    w.VloT[st] = 0.f;
  }
}

// one warp per prepended row
__global__ void __launch_bounds__(kBlock) k_negdeg_scatter(StepParams p, TableView ent, BatchView b, StepWs w) {
  const long long t = (long long)blockIdx.x * (kBlock / 32) + (threadIdx.x >> 5);
  if (t >= p.B) return;
  const int lane = threadIdx.x & 31;
  const long long c = t / p.Cs;
  const int j = (int)(t % p.Cs);
  const long long e = c * p.Cs + j;                             // the edge whose own row this is
  const long long loc = p.neg_head ? b.head_local[e] : b.tail_local[e];
  float* g = w.Bn + (c * p.Ns + j) * (long long)p.D;            // gradient of the prepended "negative" (reg'(row) included)
  float* ng = w.NG + loc * (long long)p.D;
  const float* x = row_ptr(ent, b.node_ids[loc]);
  const bool reg_on = (p.reg_coef > 0.f && p.reg_norm > 0);
  for (int v = lane; v < (p.D >> 2); v += 32) {
    float4 gv = ld4(g + 4 * v);
    if (reg_on) gv = f4_sub(gv, reg_grad4(ld4(x + 4 * v), p.reg_norm, p.reg_coef));
    red_add4(ng + 4 * v, gv);
    st4(g + 4 * v, make_float4(0.f, 0.f, 0.f, 0.f));
  }
}
}  // namespace

void launch_negdeg_ids(const LaunchCtx& c, const StepParams& p, const BatchView& b, const long long* sampled, long long* out) {
  KGE_LAUNCH(c, k_negdeg_ids, ceil_div(p.Nn, kBlock), kBlock, 0, p, b, sampled, out);
}
void launch_negdeg_zero_reg(const LaunchCtx& c, const StepParams& p, const StepWs& w) {
  KGE_LAUNCH(c, k_negdeg_zero_reg, ceil_div(p.B, kBlock), kBlock, 0, p, w);
}
void launch_negdeg_mask_scores(const LaunchCtx& c, const StepParams& p, const StepWs& w) {
  KGE_LAUNCH(c, k_negdeg_mask_scores, ceil_div(p.B, kBlock), kBlock, 0, p, w);
}
void launch_negdeg_mask_coef(const LaunchCtx& c, const StepParams& p, const StepWs& w) {
  KGE_LAUNCH(c, k_negdeg_mask_coef, ceil_div(p.B, kBlock), kBlock, 0, p, w);
}
void launch_negdeg_scatter(const LaunchCtx& c, const StepParams& p, const TableView& ent, const BatchView& b, const StepWs& w) {
  KGE_LAUNCH(c, k_negdeg_scatter, ceil_div(p.B, kBlock / 32), kBlock, 0, p, ent, b, w);
}

}  // namespace kge
