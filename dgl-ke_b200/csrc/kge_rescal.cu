// kge_rescal.cu -- RESCAL's per-edge relation-matrix work (score_fun.py:378-449).
// A relation row is a full matrix M_r [D, D] (row-major, general_models.py:232-236), so the per-edge
// work is two mat-vecs forward (M h, M t) and a rank-1 gradient + two transposed mat-vecs backward.
// One CTA per edge streams M_r exactly once per pass with 16-byte loads; warps own rows of M_r,
// lanes own column slices.  (Grouping edges by relation into a tensor-core GEMM is the next step,
// DESIGN.md "next".)
#include "kge_common.cuh"

namespace kge {


constexpr int kBlock = 256;
constexpr int kWarps = kBlock / 32;
constexpr int kMaxV = 4;            // float4 slices per lane => D <= 512

// forward: A[i] = M p (p = h in tail-corrupt mode -- the reference's transpose quirk,
// score_fun.py:445-448 -- and t in head-corrupt mode, :435), Mt[i] = M t, pos_i = h . (M t) (:387-394)
__global__ void __launch_bounds__(kBlock) k_rescal_fwd(StepParams p, const float* __restrict__ hbase,
                                                        const float* __restrict__ tbase, const float* __restrict__ rbase,
                                                        TableView ent, TableView rel, BatchView b, StepWs w,
                                                        bool dense, bool want_pos, bool want_a) {
  extern __shared__ __align__(16) float sm[];
  const int D = p.D;
  float* sh = sm;            // [D]
  float* st = sm + D;        // [D]
  float* sMh = sm + 2 * D;   // [D]
  float* sMt = sm + 3 * D;   // [D]
  __shared__ float red[kWarps];
  const long long i = blockIdx.x;
  const float *h, *t, *M;
  if (dense) {
    h = hbase + i * (long long)D; t = tbase + i * (long long)D; M = rbase + i * (long long)p.Dr;
    // kge_score_neg passes the negatives in place of the corrupted side: only the kept side is read
    if (!want_pos) { if (p.neg_head) h = t; else t = h; }
  } else {
    h = node_row(p, ent, b, w, b.head_local[i]);
    t = node_row(p, ent, b, w, b.tail_local[i]);
    M = row_ptr(rel, b.rel_ids[i]);
  }
  for (int k = threadIdx.x; k < D; k += kBlock) { sh[k] = h[k]; st[k] = t[k]; }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nv = D >> 2;
  const bool reg_on = (!dense) && (p.reg_coef > 0.f && p.reg_norm > 0);
  float reg = 0.f;
  for (int k = warp; k < D; k += kWarps) {
    const float* row = M + (long long)k * D;
    float ah = 0.f, at = 0.f;
    for (int v = lane; v < nv; v += 32) {
      float4 m4 = ld4_stream(row + 4 * v);
      ah += f4_dot(m4, ld4(sh + 4 * v));
      at += f4_dot(m4, ld4(st + 4 * v));
      if (reg_on) reg += abs_pow4_sum(m4, p.reg_norm);
    }
    ah = warp_sum(ah); at = warp_sum(at);
    if (lane == 0) { sMh[k] = ah; sMt[k] = at; }
  }
  __syncthreads();
  float pos = 0.f;
  for (int k = threadIdx.x; k < D; k += kBlock) {
    pos += sh[k] * sMt[k];
    if (want_a) {
      const float av = p.neg_head ? sMt[k] : sMh[k];
      if (w.Ahi || w.Af) {
        float hh, ll;
        split_tf32(av, hh, ll);
        const long long o = slab_off(i / p.Cs, slab_blocks(D), p.Cs, (int)(i % p.Cs), k);
        if (w.Af) w.Af[o] = av;            // fused step: k_fused<P> splits it
        else { w.Ahi[o] = hh; w.Alo[o] = ll; }
        if (w.AhiT) {
          const long long ot = slabT_off(i / p.Cs, p.Cs, D, (int)(i % p.Cs), k);
          w.AhiT[ot] = hh; w.AloT[ot] = ll;
        }
      }
      else w.A[i * (long long)D + k] = av;
    }
    if (!dense) w.Mt[i * (long long)D + k] = sMt[k];
  }
  pos = warp_sum(pos); reg = warp_sum(reg);
  if (lane == 0) red[warp] = pos;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
    for (int q = 0; q < kWarps; ++q) s += red[q];
    if (want_pos) w.pos[i] = s;
  }
  __syncthreads();
  if (reg_on) {
    if (lane == 0) red[warp] = reg;
    __syncthreads();
    if (threadIdx.x == 0) {
      float s = 0.f;
      for (int q = 0; q < kWarps; ++q) s += red[q];
      w.regp[i] = s;
    }
  } else if (!dense && threadIdx.x == 0) {
    w.regp[i] = 0.f;
  }
}

// the edge rows here, the negatives' rows by k_prep's generic blocks
int launch_rescal_prep(const LaunchCtx& c, const StepParams& p, const TableView& ent, const TableView& rel,
                       const BatchView& b, const StepWs& w) {
  size_t smem = 4 * (size_t)p.D * sizeof(float);
  KGE_LAUNCH(c, k_rescal_fwd, (unsigned)p.B, kBlock, smem, p, nullptr, nullptr, nullptr, ent, rel, b, w, false, true, true);
  return launch_prep_nonedge(c, p, ent, rel, b, w);
}

void launch_rescal_prep_dense(const LaunchCtx& c, const StepParams& p, const float* head, const float* relr,
                              const float* tail, const StepWs& w, bool want_pos, bool want_a) {
  size_t smem = 4 * (size_t)p.D * sizeof(float);
  TableView none{};
  BatchView nb{};
  KGE_LAUNCH(c, k_rescal_fwd, (unsigned)p.B, kBlock, smem, p, head, tail, relr, none, none, nb, w, true, want_pos, want_a);
}

// backward of one edge.  With u = GA_i (dL/da), g = gpos_i, p = h (tail mode) | t (head mode):
//   dL/dM[k,l] = u[k] p[l] + g h[k] t[l]   (+ reg)        -> GR[i]
//   tail mode:  dL/dh = M^T u + g (M t),   dL/dt = g M^T h
//   head mode:  dL/dt = M^T (u + g h),     dL/dh = g (M t)
__global__ void __launch_bounds__(kBlock) k_rescal_bwd(StepParams p, TableView ent, TableView rel, BatchView b, StepWs w) {
  extern __shared__ __align__(16) float sm[];
  const int D = p.D;
  float* sh = sm;             // h
  float* st = sm + D;         // t
  float* su = sm + 2 * D;     // u1: GA (tail) | GA + g h (head)
  float* sy = sm + 3 * D;     // [2][D] cross-warp accumulators for M^T u1, M^T h
  __shared__ float red[kWarps];
  const long long i = blockIdx.x;
  const long long hl = b.head_local[i], tl = b.tail_local[i], rid = b.rel_ids[i];
  const float* h = node_row(p, ent, b, w, hl);
  const float* t = node_row(p, ent, b, w, tl);
  const float* M = row_ptr(rel, rid);
  float* GR = w.GR + i * (long long)p.Dr;
  const float g = w.gpos[i];
  const float* ga = w.GA + i * (long long)D;
  for (int k = threadIdx.x; k < D; k += kBlock) {
    float hk = h[k];
    sh[k] = hk; st[k] = t[k];
    su[k] = p.neg_head ? (ga[k] + g * hk) : ga[k];
    sy[k] = 0.f; sy[D + k] = 0.f;
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nv = D >> 2;
  float4 y1[kMaxV], y2[kMaxV];
#pragma unroll
  for (int q = 0; q < kMaxV; ++q) { y1[q] = make_float4(0.f, 0.f, 0.f, 0.f); y2[q] = y1[q]; }
  float gs = 0.f;
  const float* pvec = p.neg_head ? st : sh;
  for (int k = warp; k < D; k += kWarps) {
    const float* row = M + (long long)k * D;
    const float uk = p.neg_head ? ga[k] : su[k];   // dL/da_k
    const float u1 = su[k], ghk = g * sh[k], hk = sh[k];
#pragma unroll
    for (int q = 0; q < kMaxV; ++q) {
      int v = lane + 32 * q;
      if (v < nv) {
        float4 m4 = ld4(row + 4 * v);
        float4 p4 = ld4(pvec + 4 * v), t4 = ld4(st + 4 * v);
        float4 dM = f4_add(f4_add(f4_scale(p4, uk), f4_scale(t4, ghk)), reg_grad4(m4, p.reg_norm, p.reg_coef));
        st4(GR + (long long)k * D + 4 * v, dM);
        gs += f4_dot(dM, dM);
        y1[q] = f4_fma(m4, u1, y1[q]);
        if (!p.neg_head) y2[q] = f4_fma(m4, hk, y2[q]);
      }
    }
  }
#pragma unroll
  for (int q = 0; q < kMaxV; ++q) {
    int v = lane + 32 * q;
    if (v < nv) {
      atomicAdd(&sy[4 * v + 0], y1[q].x); atomicAdd(&sy[4 * v + 1], y1[q].y);
      atomicAdd(&sy[4 * v + 2], y1[q].z); atomicAdd(&sy[4 * v + 3], y1[q].w);
      if (!p.neg_head) {
        atomicAdd(&sy[D + 4 * v + 0], y2[q].x); atomicAdd(&sy[D + 4 * v + 1], y2[q].y);
        atomicAdd(&sy[D + 4 * v + 2], y2[q].z); atomicAdd(&sy[D + 4 * v + 3], y2[q].w);
      }
    }
  }
  gs = warp_sum(gs);
  if (lane == 0) red[warp] = gs;
  __syncthreads();
  const float* mt = w.Mt + i * (long long)D;
  float* ngh = w.NG + hl * (long long)D;
  float* ngt = w.NG + tl * (long long)D;
  for (int k = threadIdx.x; k < D; k += kBlock) {
    float dh, dt;
    if (p.neg_head) { dt = sy[k]; dh = g * mt[k]; }
    else { dh = sy[k] + g * mt[k]; dt = g * sy[D + k]; }
    atomicAdd(ngh + k, dh);
    atomicAdd(ngt + k, dt);
  }
  if (threadIdx.x == 0) {
    float s = 0.f;
    for (int q = 0; q < kWarps; ++q) s += red[q];
    w.gsr[i] = s / (float)p.Dr;     // added to the relation's state_sum by the update (Adagrad phase 1)
  }
}

void launch_rescal_chain(const LaunchCtx& c, const StepParams& p, const TableView& ent, const TableView& rel,
                         const BatchView& b, const StepWs& w) {
  size_t smem = 5 * (size_t)p.D * sizeof(float);
  KGE_LAUNCH(c, k_rescal_bwd, (unsigned)p.B, kBlock, smem, p, ent, rel, b, w);
}

}  // namespace kge
