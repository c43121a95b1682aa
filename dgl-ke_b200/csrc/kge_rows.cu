// kge_rows.cu -- the row-streaming (HBM-bound) kernels of the step: one warp per embedding row,
// 16-byte vector loads, warp-shuffle reductions for the per-row dot / norm.
//
//   k_gather      ExternalEmbedding.__call__            tensor_models.py:270-302
//   k_prep        gather + edge_func + a-side of create_neg   score_fun.py:54-59,91-108,229-235,
//                 268-286,297-307,345-376,460-472,512-554 ; general_models.py:548-553
//   k_loss        LossGenerator.get_total_loss + its gradient loss.py:69-98
//   k_chain       autograd of edge_func / a-side back to h, r, t  (loss.backward(), train_pytorch.py:145)
//   k_upd_*       ExternalEmbedding.update              tensor_models.py:304-362
#include "kge_common.cuh"

namespace kge {


constexpr int kRowBlock = 256;               // 8 warps = 8 row jobs per CTA
constexpr int kWarpsPerBlock = kRowBlock / kWarp;

// ------------------------------------------------------------------------------------------ a3
__global__ void __launch_bounds__(kRowBlock) k_gather(TableView t, const long long* __restrict__ idx,
                                                       long long n, float* __restrict__ out) {
  long long job = (long long)blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
  if (job >= n) return;
  int lane = threadIdx.x & 31;
  const float* src = row_ptr(t, idx[job]);
  float* dst = out + job * (long long)t.dim;
  int nv = t.dim >> 2;
  for (int v = lane; v < nv; v += kWarp) st4(dst + 4 * v, ld4_stream(src + 4 * v));
  for (int k = (nv << 2) + lane; k < t.dim; k += kWarp) dst[k] = src[k];   // dim % 4 tail
}

void launch_gather(const LaunchCtx& c, const TableView& t, const long long* idx, long long n, float* out) {
  if (n <= 0) return;
  KGE_LAUNCH(c, k_gather, ceil_div(n, kWarpsPerBlock), kRowBlock, 0, t, idx, n, out);
}

__global__ void k_fill_zero(float* p, long long n) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  long long stride = (long long)gridDim.x * blockDim.x;
  for (; i < n; i += stride) p[i] = 0.f;
}
void launch_fill_zero(const LaunchCtx& c, float* p, long long n) {
  if (n <= 0) return;
  int grid = (int)((n + 1023) / 1024);
  if (grid > c.num_sms * 8) grid = c.num_sms * 8;
  KGE_LAUNCH(c, k_fill_zero, grid, 256, 0, p, n);
}

// ------------------------------------------------------------------------------------ a4 + a5(a)
// Per-edge model math on one 4-wide slice.  For the complex models a "slice" is 4 real parts plus
// the 4 matching imaginary parts (rows are [re | im]).
struct EdgeAcc {
  float pos;   // running sum for the positive score
  float a2;    // |a|^2 (TransE_l2)
  float reg;   // sum |r|^p
};

template <int MODEL>
__device__ __forceinline__ void edge_slice_real(float4 h, float4 r, float4 t, int neg_head, float4& a,
                                                EdgeAcc& acc) {
  if (MODEL == KGE_TRANSE_L1 || MODEL == KGE_TRANSE_L2) {
    float4 e = f4_sub(f4_add(h, r), t);
    if (MODEL == KGE_TRANSE_L2) acc.pos += f4_dot(e, e);
    else acc.pos += (fabsf(e.x) + fabsf(e.y)) + (fabsf(e.z) + fabsf(e.w));
    a = neg_head ? f4_sub(t, r) : f4_add(h, r);
    if (MODEL == KGE_TRANSE_L2) acc.a2 += f4_dot(a, a);
  } else {  // DistMult
    acc.pos += f4_hsum(f4_mul(f4_mul(h, r), t));
    a = neg_head ? f4_mul(t, r) : f4_mul(h, r);
  }
}

// complex slice: (hr,hi) head, (tr,ti) tail, (cr,ci) = relation as complex number
// (ComplEx: the row itself; RotatE: cos/sin of the phase)
template <int MODEL>
__device__ __forceinline__ void edge_slice_cplx(float4 hr, float4 hi, float4 tr, float4 ti, float4 cr, float4 ci,
                                                int neg_head, float4& are, float4& aim, EdgeAcc& acc) {
  if (MODEL == KGE_COMPLEX) {
    // score_fun.py:297-307
    float4 s = f4_sub(f4_add(f4_add(f4_mul(f4_mul(hr, tr), cr), f4_mul(f4_mul(hi, ti), cr)),
                             f4_mul(f4_mul(hr, ti), ci)),
                      f4_mul(f4_mul(hi, tr), ci));
    acc.pos += f4_hsum(s);
  } else {
    // score_fun.py:460-472
    float4 dre = f4_sub(f4_sub(f4_mul(hr, cr), f4_mul(hi, ci)), tr);
    float4 dim = f4_sub(f4_add(f4_mul(hr, ci), f4_mul(hi, cr)), ti);
    acc.pos += (sqrtf(dre.x * dre.x + dim.x * dim.x) + sqrtf(dre.y * dre.y + dim.y * dim.y)) +
               (sqrtf(dre.z * dre.z + dim.z * dim.z) + sqrtf(dre.w * dre.w + dim.w * dim.w));
  }
  if (neg_head) {   // conj(rel) * tail   (score_fun.py:353-355, 523-524)
    are = f4_add(f4_mul(tr, cr), f4_mul(ti, ci));
    aim = f4_add(f4_mul(f4_neg(tr), ci), f4_mul(ti, cr));
  } else {          // head * rel         (score_fun.py:369-371, 542-543)
    are = f4_sub(f4_mul(hr, cr), f4_mul(hi, ci));
    aim = f4_add(f4_mul(hr, ci), f4_mul(hi, cr));
  }
}

__device__ __forceinline__ void phase_cos_sin(float4 r, float inv_scale_den, float4& c, float4& s) {
  // phase = r / (emb_init / pi)   (score_fun.py:464)
  float p0 = r.x / inv_scale_den, p1 = r.y / inv_scale_den, p2 = r.z / inv_scale_den, p3 = r.w / inv_scale_den;
  sincosf(p0, &s.x, &c.x); sincosf(p1, &s.y, &c.y); sincosf(p2, &s.z, &c.z); sincosf(p3, &s.w, &c.w);
}

// One warp = one edge.  h/r/t are row pointers (table rows or dense rows).
template <int MODEL, int KIT>
__device__ __forceinline__ void edge_forward(const StepParams& p, const float* __restrict__ h,
                                             const float* __restrict__ r, const float* __restrict__ t,
                                             const RowOut& a_out, int lane, float& pos_out, float& a2_out,
                                             float& reg_out, float& nrm_out, bool want_a) {
  EdgeAcc acc{0.f, 0.f, 0.f};
  const bool reg_on = (p.reg_coef > 0.f && p.reg_norm > 0);
  // All loads of the (up to kIt) slices a lane owns are issued before any arithmetic: 9-12 independent 16-byte
  // loads in flight per lane hide HBM latency, and the longer NVLink latency when the rows live on a peer GPU.
  constexpr int kIt = KIT;                                // slices per lane loaded ahead (1: local HBM, 4: sharded)
  constexpr int kItC = KIT > 1 ? KIT / 2 : 1;             // complex models load two half-rows per slice
  const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
  if (MODEL == KGE_COMPLEX || MODEL == KGE_ROTATE) {
    const int half = p.D >> 1, nvh = half >> 2;
    const float den = p.emb_init / 3.14159265358979323846f;
    for (int v0 = 0; v0 < nvh; v0 += kWarp * kItC) {
      float4 hr[kItC], hi[kItC], tr[kItC], ti[kItC], r0[kItC], r1[kItC];
#pragma unroll
      for (int it = 0; it < kItC; ++it) {
        const int v = v0 + lane + kWarp * it;
        const bool ok = v < nvh;
        hr[it] = ok ? ld4(h + 4 * v) : z4; hi[it] = ok ? ld4(h + half + 4 * v) : z4;
        tr[it] = ok ? ld4(t + 4 * v) : z4; ti[it] = ok ? ld4(t + half + 4 * v) : z4;
        r0[it] = ok ? ld4(r + 4 * v) : z4;
        r1[it] = (ok && MODEL == KGE_COMPLEX) ? ld4(r + half + 4 * v) : z4;
      }
#pragma unroll
      for (int it = 0; it < kItC; ++it) {
        const int v = v0 + lane + kWarp * it;
        if (v >= nvh) continue;
        float4 cr, ci;
        if (MODEL == KGE_COMPLEX) {
          cr = r0[it]; ci = r1[it];
          if (reg_on) acc.reg += abs_pow4_sum(cr, p.reg_norm) + abs_pow4_sum(ci, p.reg_norm);
        } else {
          if (reg_on) acc.reg += abs_pow4_sum(r0[it], p.reg_norm);
          phase_cos_sin(r0[it], den, cr, ci);
        }
        float4 are, aim;
        edge_slice_cplx<MODEL>(hr[it], hi[it], tr[it], ti[it], cr, ci, p.neg_head, are, aim, acc);
        if (want_a) { row_store4(a_out, 4 * v, are); row_store4(a_out, half + 4 * v, aim); }
      }
    }
  } else {
    const int nv = p.D >> 2;
    for (int v0 = 0; v0 < nv; v0 += kWarp * kIt) {
      float4 h4[kIt], r4[kIt], t4[kIt];
#pragma unroll
      for (int it = 0; it < kIt; ++it) {
        const int v = v0 + lane + kWarp * it;
        const bool ok = v < nv;
        h4[it] = ok ? ld4(h + 4 * v) : z4;
        r4[it] = ok ? ld4(r + 4 * v) : z4;
        t4[it] = ok ? ld4(t + 4 * v) : z4;
      }
#pragma unroll
      for (int it = 0; it < kIt; ++it) {
        const int v = v0 + lane + kWarp * it;
        if (v >= nv) continue;
        if (reg_on) acc.reg += abs_pow4_sum(r4[it], p.reg_norm);
        float4 a;
        edge_slice_real<MODEL>(h4[it], r4[it], t4[it], p.neg_head, a, acc);
        if (want_a) row_store4(a_out, 4 * v, a);
      }
    }
  }
  float s = warp_sum(acc.pos);
  a2_out = warp_sum(acc.a2);
  reg_out = warp_sum(acc.reg);
  nrm_out = 0.f;
  if (MODEL == KGE_TRANSE_L2) { nrm_out = sqrtf(s); pos_out = p.gamma - nrm_out; }
  else if (MODEL == KGE_TRANSE_L1 || MODEL == KGE_ROTATE) pos_out = p.gamma - s;
  else pos_out = s;
}

// Job space of k_prep: one CTA per (chunk, row block) -- C * ceil(Cs/rows) blocks of edge rows, then C * ceil(Ns/rows)
// blocks of negative rows; the last block of a chunk may be partial.  One warp per row, lane -> columns as everywhere
// else.  With the wgmma engine a block is 32 rows (4 per warp, one at a time): every row is also copied to shared
// memory, and after a barrier the CTA writes the block's transposed slabs X^T[c][rb][col][0..31] from there: for each
// column one warp store of 32 rows (lane = row) is one whole 128-byte line of hi and one of lo.  Written row by row,
// each of those lines took 32 separate 4-byte stores.  Without transposed slabs (fp32 tiles) a block is 8 rows, one per
// warp, so that small batches keep every row in flight at once.
// The staging buffer (prep_stage_bytes, kge_common.cuh) is 52.5 KB at d = 400 and reaches the 227 KB a CTA may opt in
// to at d = 1792; umma_supported / fused_supported keep larger rows on the fp32 tiles, which need no transposed slabs.
__host__ __device__ inline int prep_block_rows(const StepWs& w) { return (w.AhiT || w.BhiT) ? kPrepRows : kWarpsPerBlock; }

// KIT: slices per lane loaded ahead in the negatives' rows (1: local HBM, 4: sharded table).  Those are the only rows
// k_prep may read over NVLink: with a sharded table the head / tail rows come from the local copy NC and the relation
// table is replicated, so the edge rows always take edge_forward<MODEL, 1>, which keeps the kernel within 80 registers.
template <int MODEL, int KIT>
__global__ void __launch_bounds__(kRowBlock, 3) k_prep(StepParams p, TableView ent, TableView rel, BatchView b, StepWs w,
                                                        int blk0) {
  extern __shared__ float4 prep_stage_f4[];
  float* const stage = reinterpret_cast<float*>(prep_stage_f4);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const bool reg_on = (p.reg_coef > 0.f && p.reg_norm > 0);
  const int rows = prep_block_rows(w);
  const int eblk = (p.Cs + rows - 1) / rows;
  long long blk = (long long)blk0 + blockIdx.x;
  const bool edge = blk < (long long)p.C * eblk;
  if (!edge) blk -= (long long)p.C * eblk;
  const int R = edge ? p.Cs : p.Ns, nblk = edge ? eblk : (p.Ns + rows - 1) / rows;
  const long long chunk = blk / nblk;
  const int rb = (int)(blk % nblk);
  const int nrows = min(rows, R - rb * rows);
  float* const hiT = edge ? w.AhiT : w.BhiT;
  float* const loT = edge ? w.AloT : w.BloT;
  const int S = prep_stage_stride(p.D);

  for (int rl = warp; rl < nrows; rl += kWarpsPerBlock) {   // row within the block: a partial block keeps all warps busy
    const int row = rb * rows + rl;
    float* const st = hiT ? stage + rl * S : nullptr;
    if (edge) {
      const long long job = chunk * p.Cs + row;
      const float* h = head_row(p, ent, b, w, job);     // local copies made by k_gather_nodes, or table rows
      const float* t = tail_row(p, ent, b, w, job);
      const float* r = row_ptr(rel, b.rel_ids[job]);
      float pos, a2, reg, nrm;
      // wgmma engine: A is only consumed as hi/lo operands; fused step: as fp32 slabs (split by k_fused<P>);
      // fp32 tiles: plain fp32
      const RowOut ao{(w.Ahi || w.Af) ? nullptr : w.A + job * (long long)p.D, w.Ahi, w.Alo, chunk, slab_blocks(p.D), p.Cs,
                      row, st, w.Af};
      edge_forward<MODEL, 1>(p, h, r, t, ao, lane, pos, a2, reg, nrm, true);
      if (lane == 0) {
        w.pos[job] = pos;
        if (MODEL == KGE_TRANSE_L2) { w.a2[job] = a2; w.pnorm[job] = nrm; }
        w.regp[job] = reg;
      }
    } else {
      const long long job = chunk * p.Ns + row;
      const long long ro = job * (long long)p.D;
      const float* src = w.BnRaw ? w.BnRaw + ro : row_ptr(ent, b.neg_ids[job]);   // staged by the previous step, or the table
      // fused contraction: the negatives exist only as TF32 hi/lo slabs (Bn receives their gradient later)
      const RowOut bo{p.fused ? nullptr : w.Bn + ro, w.Bhi, w.Blo, chunk, slab_blocks(p.D), p.Ns, row, st};
      float b2 = 0.f, reg = 0.f;
      const int nv = p.D >> 2;
      for (int v0 = 0; v0 < nv; v0 += kWarp * KIT) {
        float4 x[KIT];
#pragma unroll
        for (int it = 0; it < KIT; ++it) {
          const int v = v0 + lane + kWarp * it;
          x[it] = (v < nv) ? ld4_stream(src + 4 * v) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
#pragma unroll
        for (int it = 0; it < KIT; ++it) {
          const int v = v0 + lane + kWarp * it;
          if (v >= nv) continue;
          row_store4(bo, 4 * v, x[it]);
          if (MODEL == KGE_TRANSE_L2) b2 += f4_dot(x[it], x[it]);
          if (reg_on) reg += abs_pow4_sum(x[it], p.reg_norm);
        }
      }
      b2 = warp_sum(b2); reg = warp_sum(reg);
      if (lane == 0) {
        if (MODEL == KGE_TRANSE_L2) w.b2[job] = b2;
        w.regp[p.B + job] = reg;
      }
    }
  }
  if (!hiT) return;
  __syncthreads();
  // transposed slabs: warp `warp` takes column groups warp, warp + 8, ...; the padding rows of a partial block stay unwritten
  if (lane >= nrows) return;
  const long long base = ((chunk * nblk + rb) * (long long)p.D) * 32 + lane;
  const float* srow = stage + lane * S;
  for (int g = warp; g < (p.D >> 2); g += kWarpsPerBlock) {
    float4 h, l;
    split_tf32_4(*reinterpret_cast<const float4*>(srow + 4 * g), h, l);
    float* dh = hiT + base + (long long)(4 * g) * 32;
    float* dl = loT + base + (long long)(4 * g) * 32;
    dh[0] = h.x; dh[32] = h.y; dh[64] = h.z; dh[96] = h.w;
    dl[0] = l.x; dl[32] = l.y; dl[64] = l.z; dl[96] = l.w;
  }
}

// dynamic shared memory of a k_prep launch: the staging buffer exists only where the transposed slabs do (beyond 48 KB,
// d > 356, the kernel has to opt in)
size_t prep_smem(const StepWs& w, int D) { return (w.AhiT || w.BhiT) ? prep_stage_bytes(D) : 0; }

// k_prep's launch error (with whatever an earlier launch of the step left behind)
int prep_launched(int D) {
  const cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? KGE_OK : fail(KGE_ERR_CUDA, "k_prep launch (d=%d): %s", D, cudaGetErrorString(e));
}

// ExternalEmbedding.__call__ on pos_g.ndata['id'] (general_models.py:548): NC[u,:] = ent[node_ids[u],:], one warp per
// unique node, plus the node's share of the regulariser.  The only kernel (besides the negatives' gather in k_prep)
// that reads entity rows from the table -- over NVLink when the owner is a peer GPU.
template <int KIT>
__global__ void __launch_bounds__(kRowBlock) k_gather_nodes(StepParams p, TableView ent, BatchView b, StepWs w) {
  const long long u = (long long)blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
  if (u >= node_count(p)) return;
  const int lane = threadIdx.x & 31;
  const bool reg_on = (p.reg_coef > 0.f && p.reg_norm > 0);
  const float* src = row_ptr(ent, b.node_ids[u]);
  float* dst = w.NC + u * (long long)p.D;
  const int nv = p.D >> 2;
  float reg = 0.f;
  for (int v0 = 0; v0 < nv; v0 += kWarp * KIT) {
    float4 x[KIT];
#pragma unroll
    for (int it = 0; it < KIT; ++it) {
      const int v = v0 + lane + kWarp * it;
      x[it] = (v < nv) ? ld4_stream(src + 4 * v) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int it = 0; it < KIT; ++it) {
      const int v = v0 + lane + kWarp * it;
      if (v >= nv) continue;
      st4(dst + 4 * v, x[it]);
      if (reg_on) reg += abs_pow4_sum(x[it], p.reg_norm);
    }
  }
  reg = warp_sum(reg);
  if (lane == 0) w.regp[p.B + p.Nn + u] = reg;
}

void launch_gather_nodes(const LaunchCtx& c, const StepParams& p, const TableView& ent, const BatchView& b,
                         const StepWs& w) {
  if (ent.n_shards > 1) KGE_LAUNCH(c, k_gather_nodes<4>, ceil_div(p.U, kWarpsPerBlock), kRowBlock, 0, p, ent, b, w);
  else KGE_LAUNCH(c, k_gather_nodes<2>, ceil_div(p.U, kWarpsPerBlock), kRowBlock, 0, p, ent, b, w);
}

// dense-row variant: kge_score_pos (want_pos) / kge_score_neg (want_a + negatives' norms)
template <int MODEL>
__global__ void __launch_bounds__(kRowBlock) k_prep_dense(StepParams p, const float* __restrict__ head,
                                                           const float* __restrict__ relr,
                                                           const float* __restrict__ tail,
                                                           const float* __restrict__ negrows, StepWs w,
                                                           bool want_pos, bool want_a) {
  long long job = (long long)blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (job < p.B) {
    float pos, a2, reg, nrm;
    const float* hrow = head + job * (long long)p.D;
    const float* trow = tail + job * (long long)p.D;
    // kge_score_neg passes the negatives in place of the corrupted side: only the kept side is read
    if (!want_pos) { if (p.neg_head) hrow = trow; else trow = hrow; }
    const long long ro = job * (long long)p.D;
    const RowOut ao{(want_a && !w.Ahi) ? w.A + ro : nullptr, want_a ? w.Ahi : nullptr, want_a ? w.Alo : nullptr,
                    job / p.Cs, slab_blocks(p.D), p.Cs, (int)(job % p.Cs), nullptr};
    edge_forward<MODEL, 1>(p, hrow, relr + job * (long long)p.Dr, trow, ao, lane, pos, a2, reg, nrm, want_a);
    if (lane == 0) {
      if (want_pos) w.pos[job] = pos;
      if (want_a && MODEL == KGE_TRANSE_L2) w.a2[job] = a2;
    }
    return;
  }
  job -= p.B;
  if (job < p.Nn && negrows != nullptr) {
    const float* src = negrows + job * (long long)p.D;
    const long long ro = job * (long long)p.D;
    const RowOut bo{nullptr, w.Bhi, w.Blo, job / p.Ns, slab_blocks(p.D), p.Ns, (int)(job % p.Ns), nullptr};
    float b2 = 0.f;
    for (int v = lane; v < (p.D >> 2); v += kWarp) {
      float4 x = ld4(src + 4 * v);
      b2 += f4_dot(x, x);
      row_store4(bo, 4 * v, x);
    }
    b2 = warp_sum(b2);
    if (lane == 0 && MODEL == KGE_TRANSE_L2) w.b2[job] = b2;
  }
}

#define KGE_DISPATCH_MODEL(model, ...)                                      \
  switch (model) {                                                          \
    case KGE_TRANSE_L1: { constexpr int M = KGE_TRANSE_L1; __VA_ARGS__; } break; \
    case KGE_TRANSE_L2: { constexpr int M = KGE_TRANSE_L2; __VA_ARGS__; } break; \
    case KGE_DISTMULT:  { constexpr int M = KGE_DISTMULT;  __VA_ARGS__; } break; \
    case KGE_COMPLEX:   { constexpr int M = KGE_COMPLEX;   __VA_ARGS__; } break; \
    case KGE_ROTATE:    { constexpr int M = KGE_ROTATE;    __VA_ARGS__; } break; \
    default: break;                                                         \
  }

int launch_prep(const LaunchCtx& c, const StepParams& p, const TableView& ent, const TableView& rel,
                const BatchView& b, const StepWs& w) {
  const int rows = prep_block_rows(w);
  const int blocks = p.C * (ceil_div(p.Cs, rows) + ceil_div(p.Ns, rows));
  const size_t smem = prep_smem(w, p.D);
  int rc = KGE_OK;
  // sharded tables: deeper per-lane load batches hide the NVLink latency; local HBM prefers occupancy
  if (ent.n_shards > 1) {
    KGE_DISPATCH_MODEL(p.model, if (!(rc = smem_optin((const void*)k_prep<M, 4>, smem)))
                                  KGE_LAUNCH(c, (k_prep<M, 4>), blocks, kRowBlock, smem, p, ent, rel, b, w, 0));
  } else {
    KGE_DISPATCH_MODEL(p.model, if (!(rc = smem_optin((const void*)k_prep<M, 1>, smem)))
                                  KGE_LAUNCH(c, (k_prep<M, 1>), blocks, kRowBlock, smem, p, ent, rel, b, w, 0));
  }
  return rc ? rc : prep_launched(p.D);
}

int launch_prep_nonedge(const LaunchCtx& c, const StepParams& p, const TableView& ent, const TableView& rel,
                        const BatchView& b, const StepWs& w) {
  const size_t smem = prep_smem(w, p.D);
  if (int rc = smem_optin((const void*)k_prep<KGE_DISTMULT, 1>, smem)) return rc;
  const int rows = prep_block_rows(w);
  KGE_LAUNCH(c, (k_prep<KGE_DISTMULT, 1>), p.C * ceil_div(p.Ns, rows), kRowBlock, smem, p, ent, rel, b, w,
             p.C * ceil_div(p.Cs, rows));
  return prep_launched(p.D);
}

void launch_prep_dense(const LaunchCtx& c, const StepParams& p, const float* head, const float* relr,
                       const float* tail, const float* negrows, const StepWs& w, bool want_pos, bool want_a) {
  long long jobs = p.B + ((negrows && (p.model == KGE_TRANSE_L2 || w.Bhi)) ? p.Nn : 0);
  KGE_DISPATCH_MODEL(p.model, KGE_LAUNCH(c, k_prep_dense<M>, ceil_div(jobs, kWarpsPerBlock), kRowBlock, 0, p, head,
                                         relr, tail, negrows, w, want_pos, want_a));
}

// ------------------------------------------------------------------------------------------ a7
// One warp per positive i: reads its Ns negative scores, writes the backward coefficients
//   V_ij = dL/dneg_ij (bilinear, l1, RotatE)  |  dL/dneg_ij / dist_ij (TransE_l2),
// the per-row loss terms, dL/dpos_i, and (TransE_l2) sum_j V_ij.
// per-element math of k_loss: coefficient for the backward contraction + the loss term (loss.py:69-98)
struct LossRow {
  float w_i, inv2B, T, mx, den, uni;
  int adversarial, l2;
  int hinge, pairwise;
  float margin, ps, invBN;     // pairwise: the row's positive score, 1 / (B * Ns)
};
// criterion(x, label) and d/dx for label = +1 / -1 (loss.py:10-38): Hinge max(0, m - label x) -- zero gradient only where
// the term is strictly negative (`loss[loss < 0] = 0`); Logsigmoid / Logistic / BCE softplus(-label x)
__device__ __forceinline__ float crit(const LossRow& r, float x, float label, float& dx) {
  if (r.hinge) {
    const float t = r.margin - label * x;
    dx = (t < 0.f) ? 0.f : -label;
    return fmaxf(t, 0.f);
  }
  dx = -label * sigmoidf(-label * x);
  return softplusf(-label * x);
}
__device__ __forceinline__ float loss_elem(const LossRow& r, float sc, float dist, float& nls, float& rs, float& gp) {
  float g;
  if (r.pairwise) {
    float dd;
    const float l = crit(r, r.ps - sc, 1.f, dd);           // criterion(pos_i - neg_ij, 1) * w_i, mean over all pairs
    nls += l * r.w_i * r.uni;
    g = -dd * r.w_i * r.invBN;                               // dL/dneg_ij
    gp += dd * r.w_i * r.invBN;                              // dL/dpos_i, summed over j by the caller
  } else {
    const float pij = r.adversarial ? expf(sc * r.T - r.mx) / r.den : r.uni;
    float dd;
    const float l = crit(r, sc, -1.f, dd);
    nls += pij * (l * r.w_i);
    g = pij * dd * r.w_i * r.inv2B;                          // dL/dneg_ij
  }
  float coef = g;
  // dist = |a-b| from the score kernel; a clamped distance (sq <= 1e-30) has zero gradient in the reference (clamp_min_)
  if (r.l2) { coef = (dist > 1.5e-15f) ? g / dist : 0.f; rs += coef; }
  return coef;
}

__global__ void __launch_bounds__(kRowBlock) k_loss(StepParams p, const float* __restrict__ pos,
                                                     const float* __restrict__ S, const float* __restrict__ wt,
                                                     const float* __restrict__ wbar, float* __restrict__ V,
                                                     float* __restrict__ gpos, float* __restrict__ rowsum,
                                                     float* __restrict__ pl, float* __restrict__ nl,
                                                     float* __restrict__ Vhi, float* __restrict__ Vlo,
                                                     float* __restrict__ VhiT, float* __restrict__ VloT) {
  long long i = (long long)blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
  if (i >= p.B) return;
  const int lane = threadIdx.x & 31;
  const float* s = S + i * (long long)p.Ns;
  float* v = V + i * (long long)p.Ns;
  LossRow r;
  r.w_i = wt ? wt[i] : 1.f;
  r.inv2B = 0.5f / (float)p.B;
  r.T = p.adv_temperature; r.mx = -INFINITY; r.den = 1.f; r.uni = 1.f / (float)p.Ns;
  r.adversarial = p.adversarial && !p.pairwise; r.l2 = (p.model == KGE_TRANSE_L2);
  r.hinge = p.hinge; r.pairwise = p.pairwise; r.margin = p.margin;
  r.ps = pos[i]; r.invBN = 1.f / ((float)p.B * (float)p.Ns);
  float gp = 0.f;
  const long long chunk = i / p.Cs;
  const int il = (int)(i % p.Cs), nblk = slab_blocks(p.Ns);
  float nls = 0.f, rs = 0.f;
  if (p.Ns <= 8 * kWarp) {
    // row in registers: every global load of the row is issued up front, the three passes run on registers
    float sc[8], ds[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const int j = lane + kWarp * q;
      sc[q] = (j < p.Ns) ? s[j] : -INFINITY;
      ds[q] = (r.l2 && j < p.Ns) ? v[j] : 1.f;
    }
    if (r.adversarial) {
      float mx = -INFINITY;
#pragma unroll
      for (int q = 0; q < 8; ++q) mx = fmaxf(mx, sc[q] * r.T);     // padding contributes -inf
      r.mx = warp_max(mx);
      float d = 0.f;
#pragma unroll
      for (int q = 0; q < 8; ++q) if (lane + kWarp * q < p.Ns) d += expf(sc[q] * r.T - r.mx);
      r.den = warp_sum(d);
    }
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const int j = lane + kWarp * q;
      if (j >= p.Ns) continue;
      const float coef = loss_elem(r, sc[q], ds[q], nls, rs, gp);
      v[j] = coef;
      if (Vhi) {
        float hh, ll;
        split_tf32(coef, hh, ll);
        const long long o = slab_off(chunk, nblk, p.Cs, il, j);
        Vhi[o] = hh; Vlo[o] = ll;
        const long long ot = slabT_off(chunk, p.Cs, p.Ns, il, j);
        VhiT[ot] = hh; VloT[ot] = ll;
      }
    }
  } else {
    if (r.adversarial) {
      float mx = -INFINITY;
      for (int j = lane; j < p.Ns; j += kWarp) mx = fmaxf(mx, s[j] * r.T);
      r.mx = warp_max(mx);
      float d = 0.f;
      for (int j = lane; j < p.Ns; j += kWarp) d += expf(s[j] * r.T - r.mx);
      r.den = warp_sum(d);
    }
    for (int j = lane; j < p.Ns; j += kWarp) {
      const float coef = loss_elem(r, s[j], r.l2 ? v[j] : 1.f, nls, rs, gp);
      v[j] = coef;
      if (Vhi) {
        float hh, ll;
        split_tf32(coef, hh, ll);
        const long long o = slab_off(chunk, nblk, p.Cs, il, j);
        Vhi[o] = hh; Vlo[o] = ll;
        const long long ot = slabT_off(chunk, p.Cs, p.Ns, il, j);
        VhiT[ot] = hh; VloT[ot] = ll;
      }
    }
  }
  nls = warp_sum(nls);
  rs = warp_sum(rs);
  gp = warp_sum(gp);
  if (lane == 0) {
    float ps = pos[i];
    float wb = wt ? *wbar : 1.f;        // loss.py:75,82: [B] * [B,1] -> mean(pl) * mean(w)
    if (p.pairwise) {                   // one term per (i, j) pair; no separate positive loss
      pl[i] = 0.f;
      gpos[i] = gp;
    } else {
      float dd;
      pl[i] = crit(r, ps, 1.f, dd);
      gpos[i] = dd * wb * r.inv2B;
    }
    nl[i] = nls;
    if (r.l2) rowsum[i] = rs;
  }
}

// colsum[c, j] = sum_i V[c, i, j]: one CTA per (chunk, 32 columns); 8 warps split the rows, fixed-order
// shared-memory reduction (deterministic).
__global__ void __launch_bounds__(256) k_colsum(StepParams p, const float* __restrict__ V, float* __restrict__ colsum) {
  __shared__ float part[8][33];
  const int c = blockIdx.y, j = blockIdx.x * 32 + (threadIdx.x & 31), w = threadIdx.x >> 5;
  float s = 0.f;
  if (j < p.Ns) {
    const float* v = V + ((long long)c * p.Cs) * p.Ns + j;
    for (int i = w; i < p.Cs; i += 8) s += v[(long long)i * p.Ns];
  }
  part[w][threadIdx.x & 31] = s;
  __syncthreads();
  if (w == 0 && j < p.Ns) {
    float t = 0.f;
#pragma unroll
    for (int q = 0; q < 8; ++q) t += part[q][threadIdx.x];
    colsum[(long long)c * p.Ns + j] = t;
  }
}

__device__ __forceinline__ float block_sum(float v, float* sh) {
  v = warp_sum(v);
  int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  __syncthreads();
  if (l == 0) sh[w] = v;
  __syncthreads();
  float r = (threadIdx.x < (blockDim.x >> 5)) ? sh[threadIdx.x] : 0.f;
  if (w == 0) r = warp_sum(r);
  return r;   // valid in warp 0
}

__global__ void __launch_bounds__(1024) k_mean(const float* __restrict__ x, long long n, float* __restrict__ out) {
  __shared__ float sh[32];
  float s = 0.f;
  for (long long i = threadIdx.x; i < n; i += blockDim.x) s += x[i];
  s = block_sum(s, sh);
  if (threadIdx.x == 0) *out = s / (float)n;
}

// log4 = {pos_loss, neg_loss, loss (no reg), reg}.  kRedBlocks CTAs reduce fixed slices into partials;
// the CTA that finishes last (ticket counter) adds the partials in index order => deterministic.
constexpr int kRedBlocks = 64;
__device__ void reduce_log_part(const StepParams& p, const StepWs& w, long long nreg, const float* wbar, float* log4,
                                int bid, int nb) {
  __shared__ float sh[32];
  __shared__ bool last;
  const float *pl = w.pl, *nl = w.nl, *regp = w.regp;
  float* partial = w.red_partial;
  unsigned int* ticket = w.red_ticket;
  float a = 0.f, b = 0.f, r = 0.f;
  const long long t0 = (long long)bid * blockDim.x + threadIdx.x, stride = (long long)nb * blockDim.x;
  for (long long i = t0; i < p.B; i += stride) { a += pl[i]; b += nl[i]; }
  for (long long i = t0; i < nreg; i += stride) r += regp[i];
  a = block_sum(a, sh);
  b = block_sum(b, sh);
  r = block_sum(r, sh);
  if (threadIdx.x == 0) {
    partial[bid * 3 + 0] = a; partial[bid * 3 + 1] = b; partial[bid * 3 + 2] = r;
    __threadfence();
    unsigned int t = atomicAdd(ticket, 1u);
    last = (t == (unsigned int)nb - 1);
  }
  __syncthreads();
  if (last) {
    __threadfence();
    // fixed-order tree over the partials (one per thread), deterministic
    float sa = 0.f, sb = 0.f, sr = 0.f;
    if ((int)threadIdx.x < nb) {
      sa = ((volatile float*)partial)[threadIdx.x * 3 + 0];
      sb = ((volatile float*)partial)[threadIdx.x * 3 + 1];
      sr = ((volatile float*)partial)[threadIdx.x * 3 + 2];
    }
    sa = block_sum(sa, sh);
    sb = block_sum(sb, sh);
    sr = block_sum(sr, sh);
    if (threadIdx.x == 0) {
      float pos_loss = sa / (float)p.B * (wbar ? *wbar : 1.f);
      float neg_loss = sb / (float)p.B;
      // pairwise (loss.py:76-80): the mean over all pairs IS the loss, and the log holds no pos_loss / neg_loss
      log4[0] = p.pairwise ? 0.f : pos_loss; log4[1] = p.pairwise ? 0.f : neg_loss;
      log4[2] = p.pairwise ? neg_loss : (neg_loss + pos_loss) / 2.f;
      log4[3] = p.reg_coef * sr;
      *ticket = 0u;      // ready for the next step
    }
  }
}

// log4 = {pos_loss, neg_loss, loss (no reg), reg}.  kRedBlocks CTAs reduce fixed slices into partials;
// the CTA that finishes last (ticket counter) adds the partials in index order => deterministic.
__global__ void __launch_bounds__(256) k_reduce_log(StepParams p, StepWs w, long long nreg, const float* __restrict__ wbar,
                                                     float* __restrict__ log4) {
  if (nreg > 0 && p.U_dev) nreg = p.B + p.Nn + *p.U_dev;
  reduce_log_part(p, w, nreg, wbar, log4, blockIdx.x, gridDim.x);
}

void launch_wbar(const LaunchCtx& c, const StepParams& p, const float* wt, const StepWs& w) {
  if (wt) KGE_LAUNCH(c, k_mean, 1, 1024, 0, wt, p.B, w.wbar);
}

void launch_reduce_log(const LaunchCtx& c, const StepParams& p, const float* wt, const StepWs& w, float* log4,
                       bool want_reg) {
  const bool reg_on = want_reg && (p.reg_coef > 0.f && p.reg_norm > 0);
  if (log4)
    KGE_LAUNCH(c, k_reduce_log, kRedBlocks, 256, 0, p, w, reg_on ? (p.B + p.Nn + p.U) : 0, wt ? w.wbar : nullptr, log4);
}

void launch_loss_rows(const LaunchCtx& c, const StepParams& p, const float* pos, const float* S, const float* wt,
                      const StepWs& w) {
  KGE_LAUNCH(c, k_loss, ceil_div(p.B, kWarpsPerBlock), kRowBlock, 0, p, pos, S, wt, w.wbar, w.V, w.gpos, w.rowsum,
             w.pl, w.nl, w.Vhi, w.Vlo, w.VhiT, w.VloT);
}

void launch_colsum(const LaunchCtx& c, const StepParams& p, const StepWs& w) {
  if (p.model == KGE_TRANSE_L2) KGE_LAUNCH(c, k_colsum, dim3(ceil_div(p.Ns, 32), p.C), 256, 0, p, w.V, w.colsum);
}

void launch_loss(const LaunchCtx& c, const StepParams& p, const float* pos, const float* S, const float* wt,
                 const StepWs& w, float* log4, bool want_reg) {
  launch_wbar(c, p, wt, w);
  launch_loss_rows(c, p, pos, S, wt, w);
  launch_colsum(c, p, w);
  launch_reduce_log(c, p, wt, w, log4, want_reg);
}

// ------------------------------------------------------------------------------------------ a9
// One warp per edge: autograd of edge_func and of the a-side, given GA = dL/da (from the
// contraction kernels) and gpos = dL/dpos.  Emits
//   NG[head_local] += dL/dh,  NG[tail_local] += dL/dt          (red.add, L2-resident workspace)
//   GR[i] = dL/dr_i + reg'(r_i),  rel.state_sum[rel_id] += mean(GR[i]^2)   (Adagrad phase 1, a10)
template <int MODEL, int KIT>
__global__ void __launch_bounds__(kRowBlock) k_chain(StepParams p, TableView ent, TableView rel, BatchView b, StepWs w) {
  const long long i = (long long)blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
  if (i >= p.B) return;
  const int lane = threadIdx.x & 31;
  const long long hl = b.head_local[i], tl = b.tail_local[i], rid = b.rel_ids[i];
  const float* h = head_row(p, ent, b, w, i);
  const float* t = tail_row(p, ent, b, w, i);
  const float* r = row_ptr(rel, rid);
  const float* ga = w.GA + i * (long long)p.D;
  float* ngh = w.NG + hl * (long long)p.D;
  float* ngt = w.NG + tl * (long long)p.D;
  // relation gradient: its own row per edge (what the reference traces), or summed per relation (fused step)
  float* gr = p.rel_dense ? (w.rg + rid * (long long)p.Dr) : (w.GR + i * (long long)p.Dr);
  const bool dense = p.rel_dense != 0;
  auto rel_out = [&](int col, float4 v) { if (dense) red_add4(gr + col, v); else st4(gr + col, v); };
  const float gp = w.gpos[i];
  float gs = 0.f;

  if (MODEL == KGE_COMPLEX || MODEL == KGE_ROTATE) {
    const int half = p.D >> 1, nvh = half >> 2;
    const float den = p.emb_init / 3.14159265358979323846f;
    for (int v = lane; v < nvh; v += kWarp) {
      float4 hr = ld4(h + 4 * v), hi = ld4(h + half + 4 * v);
      float4 tr = ld4(t + 4 * v), ti = ld4(t + half + 4 * v);
      float4 gre = ld4(ga + 4 * v), gim = ld4(ga + half + 4 * v);
      float4 cr, ci, ph;
      if (MODEL == KGE_COMPLEX) { cr = ld4(r + 4 * v); ci = ld4(r + half + 4 * v); }
      else { ph = ld4(r + 4 * v); phase_cos_sin(ph, den, cr, ci); }
      float4 dhr, dhi, dtr, dti, dcr, dci;   // d/d(head), d/d(tail), d/d(rel as complex)
      if (MODEL == KGE_COMPLEX) {
        // pos = sum hr*tr*cr + hi*ti*cr + hr*ti*ci - hi*tr*ci
        dhr = f4_scale(f4_add(f4_mul(tr, cr), f4_mul(ti, ci)), gp);
        dhi = f4_scale(f4_sub(f4_mul(ti, cr), f4_mul(tr, ci)), gp);
        dtr = f4_scale(f4_sub(f4_mul(hr, cr), f4_mul(hi, ci)), gp);
        dti = f4_scale(f4_add(f4_mul(hi, cr), f4_mul(hr, ci)), gp);
        dcr = f4_scale(f4_add(f4_mul(hr, tr), f4_mul(hi, ti)), gp);
        dci = f4_scale(f4_sub(f4_mul(hr, ti), f4_mul(hi, tr)), gp);
      } else {
        // pos = gamma - sum sqrt(dre^2 + dim^2)
        float4 dre = f4_sub(f4_sub(f4_mul(hr, cr), f4_mul(hi, ci)), tr);
        float4 dim = f4_sub(f4_add(f4_mul(hr, ci), f4_mul(hi, cr)), ti);
        float4 qre, qim;
#define KGE_Q(c_)                                                                    \
        { float m = sqrtf(dre.c_ * dre.c_ + dim.c_ * dim.c_); float s_ = (m > 0.f) ? (-gp / m) : 0.f; \
          qre.c_ = dre.c_ * s_; qim.c_ = dim.c_ * s_; }
        KGE_Q(x) KGE_Q(y) KGE_Q(z) KGE_Q(w)
#undef KGE_Q
        dhr = f4_add(f4_mul(qre, cr), f4_mul(qim, ci));
        dhi = f4_sub(f4_mul(qim, cr), f4_mul(qre, ci));
        dtr = f4_neg(qre);
        dti = f4_neg(qim);
        dcr = f4_add(f4_mul(qre, hr), f4_mul(qim, hi));
        dci = f4_sub(f4_mul(qim, hr), f4_mul(qre, hi));
      }
      if (p.neg_head) {   // a = conj(c) * t
        dtr = f4_add(dtr, f4_sub(f4_mul(gre, cr), f4_mul(gim, ci)));
        dti = f4_add(dti, f4_add(f4_mul(gre, ci), f4_mul(gim, cr)));
        dcr = f4_add(dcr, f4_add(f4_mul(gre, tr), f4_mul(gim, ti)));
        dci = f4_add(dci, f4_sub(f4_mul(gre, ti), f4_mul(gim, tr)));
      } else {            // a = h * c
        dhr = f4_add(dhr, f4_add(f4_mul(gre, cr), f4_mul(gim, ci)));
        dhi = f4_add(dhi, f4_sub(f4_mul(gim, cr), f4_mul(gre, ci)));
        dcr = f4_add(dcr, f4_add(f4_mul(gre, hr), f4_mul(gim, hi)));
        dci = f4_add(dci, f4_sub(f4_mul(gim, hr), f4_mul(gre, hi)));
      }
      red_add4(ngh + 4 * v, dhr); red_add4(ngh + half + 4 * v, dhi);
      red_add4(ngt + 4 * v, dtr); red_add4(ngt + half + 4 * v, dti);
      if (MODEL == KGE_COMPLEX) {
        float4 g0 = f4_add(dcr, reg_grad4(cr, p.reg_norm, p.reg_coef));
        float4 g1 = f4_add(dci, reg_grad4(ci, p.reg_norm, p.reg_coef));
        rel_out(4 * v, g0); rel_out(half + 4 * v, g1);
        gs += f4_dot(g0, g0) + f4_dot(g1, g1);
      } else {
        // d/dphase = -dc*sin + ds*cos ; d/dr = d/dphase / (emb_init/pi)
        float4 dth = f4_sub(f4_mul(dci, cr), f4_mul(dcr, ci));
        float4 g0 = make_float4(dth.x / den, dth.y / den, dth.z / den, dth.w / den);
        g0 = f4_add(g0, reg_grad4(ph, p.reg_norm, p.reg_coef));
        rel_out(4 * v, g0);
        gs += f4_dot(g0, g0);
      }
    }
  } else {
    const int nv = p.D >> 2;
    float nrm_scale = 0.f, rsum = 0.f;
    if (MODEL == KGE_TRANSE_L2) {
      float n = w.pnorm[i];                  // |h + r - t| as computed by the forward
      nrm_scale = (n > 0.f) ? (-gp / n) : 0.f;
      rsum = w.rowsum[i];
    }
    const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int v0 = 0; v0 < nv; v0 += kWarp * KIT) {
      // 4*KIT independent 16-byte loads per lane before any arithmetic (HBM / NVLink latency hiding)
      float4 hq[KIT], rq[KIT], tq[KIT], gq[KIT];
#pragma unroll
      for (int it = 0; it < KIT; ++it) {
        const int v = v0 + lane + kWarp * it;
        const bool ok = v < nv;
        hq[it] = ok ? ld4(h + 4 * v) : z4; rq[it] = ok ? ld4(r + 4 * v) : z4;
        tq[it] = ok ? ld4(t + 4 * v) : z4; gq[it] = ok ? ld4(ga + 4 * v) : z4;
      }
#pragma unroll
      for (int it = 0; it < KIT; ++it) {
        const int v = v0 + lane + kWarp * it;
        if (v >= nv) continue;
        const float4 h4 = hq[it], r4 = rq[it], t4 = tq[it], g4 = gq[it];
        float4 dh, dt, dr;
        if (MODEL == KGE_TRANSE_L1 || MODEL == KGE_TRANSE_L2) {
          float4 e = f4_sub(f4_add(h4, r4), t4);
          float4 u;   // gpos * dpos/dh
          if (MODEL == KGE_TRANSE_L2) u = f4_scale(e, nrm_scale);
          else u = make_float4(-gp * sgnf(e.x), -gp * sgnf(e.y), -gp * sgnf(e.z), -gp * sgnf(e.w));
          float4 a = p.neg_head ? f4_sub(t4, r4) : f4_add(h4, r4);
          float4 gA = (MODEL == KGE_TRANSE_L2) ? f4_fma(a, -rsum, g4) : g4;   // GA - rowsum * a
          if (p.neg_head) { dt = f4_sub(gA, u); dr = f4_sub(u, gA); dh = u; }
          else            { dh = f4_add(u, gA); dr = dh; dt = f4_neg(u); }
        } else {  // DistMult
          dh = f4_scale(f4_mul(r4, t4), gp);
          dr = f4_scale(f4_mul(h4, t4), gp);
          dt = f4_scale(f4_mul(h4, r4), gp);
          if (p.neg_head) { dt = f4_add(dt, f4_mul(g4, r4)); dr = f4_add(dr, f4_mul(g4, t4)); }
          else            { dh = f4_add(dh, f4_mul(g4, r4)); dr = f4_add(dr, f4_mul(g4, h4)); }
        }
        red_add4(ngh + 4 * v, dh);
        red_add4(ngt + 4 * v, dt);
        dr = f4_add(dr, reg_grad4(r4, p.reg_norm, p.reg_coef));
        rel_out(4 * v, dr);
        gs += f4_dot(dr, dr);
      }
    }
  }
  // mean(g^2) of this edge's relation row: added to state_sum by the update (Adagrad phase 1), never here
  gs = warp_sum(gs);
  if (lane == 0) {
    if (dense) atomicAdd(w.rgs + rid, gs / (float)p.Dr);
    else w.gsr[i] = gs / (float)p.Dr;
  }
}

void launch_chain(const LaunchCtx& c, const StepParams& p, const TableView& ent, const TableView& rel,
                  const BatchView& b, const StepWs& w) {
  if (ent.n_shards > 1) {
    KGE_DISPATCH_MODEL(p.model, KGE_LAUNCH(c, (k_chain<M, 4>), ceil_div(p.B, kWarpsPerBlock), kRowBlock, 0, p, ent, rel, b, w));
  } else {
    KGE_DISPATCH_MODEL(p.model, KGE_LAUNCH(c, (k_chain<M, 1>), ceil_div(p.B, kWarpsPerBlock), kRowBlock, 0, p, ent, rel, b, w));
  }
}

// ------------------------------------------------------------------------------------------ a10
// ExternalEmbedding.update (tensor_models.py:304-362) of the step's trace entries, as ONE kernel of three phases
// separated by grid barriers (cooperative launch: every CTA is resident), or as three launches of one phase each:
//
//   phase 1  entity entry 1: the unique positive nodes.  Indices are unique => state and row are updated by the
//            same warp without atomics (across GPUs: system-scope atomics).  Re-zeroes NG.  Also the dense
//            per-relation Adagrad of the fused step (rel_dense: unique rows as well).
//   phase 2  Adagrad phase 1 of the entries with possibly duplicated indices: state_sum[idx] += mean(g^2) for every
//            row of entity entry 2 (negatives) and of the relation entry (per edge).
//   phase 3  their phase 2: emb[idx] += -lr * g / (sqrt(state_sum[idx]) + 1e-10), then (fused step) the log scalars.
//
// The barriers reproduce the reference's order: entry 1 completes before entry 2 adds to state_sum; inside an entry
// every state add lands before any row is scaled.
struct UpdArgs {
  StepParams p;
  TableView ent, rel;
  BatchView b;
  StepWs w;
  float* log4;          // non-null: phase 3 also reduces {pos_loss, neg_loss, loss, reg}
  const float* wt;      // edge weights (for the log scalars) or null
  int phase_lo, phase_hi;
  int bulk_red;         // row scatters as bulk reductions (UBLKRED) instead of per-lane red.add
};

__device__ __forceinline__ unsigned int ld_acquire_u32(const unsigned int* p) {
  unsigned int v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
// all CTAs of the (co-resident) grid; ctr is zero on entry and is left at gridDim.x
__device__ __forceinline__ void grid_barrier(unsigned int* ctr) {
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    atomicAdd(ctr, 1u);
    while (ld_acquire_u32(ctr) < gridDim.x) __nanosleep(200);
    __threadfence();
  }
  __syncthreads();
}

// Row scatter as ONE bulk reduction (cp.reduce.async.bulk ... add.f32, SASS UBLKRED): the warp writes the scaled
// gradient row to a shared-memory staging buffer and an elected lane hands it to the copy engine, which adds it into the
// table row -- in this GPU's L2 or, for a peer's row, over NVLink in large packets instead of one 16-byte red.add per
// lane (100 per 1600-B row).  Two buffers per warp: the reduction of row i reads one while row i+1 is staged in the other.
constexpr int kRedRowFloats = 512;
struct RedStage {
  float* buf;           // the warp's two buffers of kRedRowFloats, back to back; null: per-lane red.add instead
  unsigned n;           // rows issued by this warp
};
__device__ __forceinline__ float* red_stage_buf(const RedStage& r) { return r.buf + (r.n & 1u) * kRedRowFloats; }
__device__ __forceinline__ float* red_stage_acquire(RedStage& r, int lane) {
  // the bulk group issued two rows ago read this buffer: all but the newest group must have finished reading
  if (lane == 0) asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");
  __syncwarp();
  return red_stage_buf(r);
}
__device__ __forceinline__ void red_stage_issue(RedStage& r, float* dst, int dim, int lane) {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");      // generic-proxy writes -> visible to the async proxy
  __syncwarp();
  if (lane == 0) {
    asm volatile("cp.reduce.async.bulk.global.shared::cta.bulk_group.add.f32 [%0], [%1], %2;"
                 :: "l"(dst), "r"((unsigned)__cvta_generic_to_shared(red_stage_buf(r))), "r"((unsigned)dim * 4u) : "memory");
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
  }
  ++r.n;
}
__device__ __forceinline__ void red_stage_drain(int lane) {
  if (lane == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
  __syncwarp();
}
__device__ __forceinline__ void st_shared4(float* p, float4 v) { *reinterpret_cast<float4*>(p) = v; }

// state_sum[id] += gs of a row with a unique index, by lane 0; returns the new state in every lane.  On one GPU lane 0
// loaded the old value st_old together with the row; across GPUs the add is a system-scope atomic, because other GPUs
// may add to the same state.
__device__ __forceinline__ float upd_state(float* st, float st_old, float gs, bool sharded, int lane) {
  float s_new = 0.f;
  if (lane == 0) {
    if (sharded) s_new = atomicAdd_system(st, gs) + gs;
    else { s_new = st_old + gs; *st = s_new; }
  }
  return __shfl_sync(0xffffffffu, s_new, 0);
}

// id = node_ids[u], loaded by the caller one job ahead.  On one GPU the state scalar is loaded together with the row: its
// address depends only on the id, so the node costs one memory round trip before its stores.
__device__ __forceinline__ void upd_node(const StepParams& p, const TableView& ent, const BatchView& b, const StepWs& w,
                                         long long u, long long id, int lane, RedStage& rs) {
  float* row = row_ptr(ent, id);
  float* ng = w.NG + u * (long long)p.D;
  const float* nc = p.use_nc ? (w.NC + u * (long long)p.D) : row;   // the traced copy of the row (node_row)
  const int nv = p.D >> 2;
  const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
  const bool sharded = ent.n_shards > 1;
  const bool reg_on = (p.reg_coef > 0.f && p.reg_norm > 0);
  float* st = state_ptr(ent, id);
  const float st_old = (!sharded && lane == 0) ? *st : 0.f;
  if (nv <= 4 * kWarp) {
    // D <= 512: all of the row's loads (NG and the traced copy) are issued before any arithmetic, and the sums stay in
    // registers for the second half -- one trip through memory and 8 independent 16-byte loads in flight per lane
    float4 x[4], gq[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int v = lane + kWarp * q;
      x[q] = (v < nv) ? ld4(nc + 4 * v) : z;
      gq[q] = (v < nv) ? ld4(ng + 4 * v) : z;
    }
    float gs = 0.f, reg = 0.f;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      gq[q] = f4_add(gq[q], reg_grad4(x[q], p.reg_norm, p.reg_coef));     // padding lanes: 0 + reg'(0) = 0
      gs += f4_dot(gq[q], gq[q]);
      if (reg_on && node_reg_in_update(p)) reg += abs_pow4_sum(x[q], p.reg_norm);
    }
    gs = warp_sum(gs) / (float)p.D;
    if (node_reg_in_update(p)) {            // no k_gather_nodes ran: this node's share of the regulariser is produced here
      reg = warp_sum(reg);
      if (lane == 0) w.regp[p.B + p.Nn + u] = reg;
    }
    const float s_new = upd_state(st, st_old, gs, sharded, lane);
    const float nlr_std = -p.lr / (sqrtf(s_new) + 1e-10f);
    float* stage = (sharded && rs.buf) ? red_stage_acquire(rs, lane) : nullptr;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int v = lane + kWarp * q;
      if (v < nv) {
        if (stage) st_shared4(stage + 4 * v, f4_scale(gq[q], nlr_std));
        else if (sharded) red_add4_sys(row + 4 * v, f4_scale(gq[q], nlr_std));
        else st4(row + 4 * v, f4_fma(gq[q], nlr_std, x[q]));
        st4(ng + 4 * v, z);
      }
    }
    if (stage) red_stage_issue(rs, row, p.D, lane);
    return;
  }
  // pass 1: g = NG + reg'(x), mean(g^2)
  float gs = 0.f, reg = 0.f;
  for (int v = lane; v < nv; v += kWarp) {
    const float4 x = ld4(nc + 4 * v);
    float4 g = f4_add(ld4(ng + 4 * v), reg_grad4(x, p.reg_norm, p.reg_coef));
    gs += f4_dot(g, g);
    if (reg_on && node_reg_in_update(p)) reg += abs_pow4_sum(x, p.reg_norm);
  }
  gs = warp_sum(gs) / (float)p.D;
  if (node_reg_in_update(p)) {            // no k_gather_nodes ran: this node's share of the regulariser is produced here
    reg = warp_sum(reg);
    if (lane == 0) w.regp[p.B + p.Nn + u] = reg;
  }
  const float s_new = upd_state(st, st_old, gs, sharded, lane);
  const float stdv = sqrtf(s_new) + 1e-10f;
  const float nlr_std = -p.lr / stdv;
  // pass 2: emb[id] += -lr * g / std.  Indices are unique, so on one GPU the new row is (traced copy + step);
  // across GPUs the step is a system-scope red.add (atomic w.r.t. peers).
  for (int v = lane; v < nv; v += kWarp) {
    float4 x = ld4(nc + 4 * v);
    float4 g = f4_add(ld4(ng + 4 * v), reg_grad4(x, p.reg_norm, p.reg_coef));
    const float4 tmp = f4_scale(g, nlr_std);       // (-lr * g) / std up to one rounding: one division per row, not per element
    if (sharded) red_add4_sys(row + 4 * v, tmp);
    else st4(row + 4 * v, f4_add(x, tmp));
    st4(ng + 4 * v, z);
  }
}

// state_sum[r] += gs by lane 0, then the relation's sum is re-zeroed once every lane has read it
__device__ __forceinline__ float upd_rel_state(float* st, float st_old, float gs, float* gs_src, int lane) {
  float s_new = 0.f;
  if (lane == 0) { s_new = st_old + gs; *st = s_new; }
  s_new = __shfl_sync(0xffffffffu, s_new, 0);
  __syncwarp();
  if (lane == 0) *gs_src = 0.f;
  return s_new;
}
// dense per-relation Adagrad (unique rows): summing the occurrences first is the same math as
// ExternalEmbedding.update, every occurrence is scaled by the same final state (tensor_models.py:352-361).
// Up to 512 columns, the sum, the state and both rows are loaded at once: one memory round trip per relation.
__device__ __forceinline__ void upd_rel_dense(const TableView& rel, float* rg, float* rgs, long long r, float lr, int lane) {
  float* st = state_ptr(rel, r);
  float* row = row_ptr(rel, r);
  float* g = rg + r * (long long)rel.dim;
  const int nv = rel.dim >> 2;
  const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
  const float gs = rgs[r], st_old = (lane == 0) ? *st : 0.f;
  if (nv <= 4 * kWarp) {
    float4 x[4], e[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int v = lane + kWarp * q;
      x[q] = (v < nv) ? ld4(g + 4 * v) : z;
      e[q] = (v < nv) ? ld4(row + 4 * v) : z;
    }
    if (gs == 0.f) return;         // relation not touched this step
    const float s_new = upd_rel_state(st, st_old, gs, rgs + r, lane);
    const float stdv = sqrtf(s_new) + 1e-10f;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int v = lane + kWarp * q;
      if (v < nv) { st4(row + 4 * v, f4_fma(x[q], -lr / stdv, e[q])); st4(g + 4 * v, z); }
    }
    return;
  }
  if (gs == 0.f) return;
  const float s_new = upd_rel_state(st, st_old, gs, rgs + r, lane);
  const float stdv = sqrtf(s_new) + 1e-10f;
  for (int v = lane; v < nv; v += kWarp) {
    float4 x = ld4(g + 4 * v), e = ld4(row + 4 * v);
    st4(row + 4 * v, f4_fma(x, -lr / stdv, e));
    st4(g + 4 * v, z);
  }
}

__device__ __forceinline__ void apply_row(const TableView& t, long long id, const float* g, int dim, float lr, int lane,
                                          RedStage& rs) {
  float* row = row_ptr(t, id);
  const int nv = dim >> 2;
  if (nv <= 4 * kWarp && (dim & 3) == 0) {
    // all loads of the gradient row in flight before the state scalar is needed
    float4 x[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int v = lane + kWarp * q;
      x[q] = (v < nv) ? ld4(g + 4 * v) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
    const float nlr_std = -lr / (sqrtf(*state_ptr(t, id)) + 1e-10f);
    if (rs.buf) {
      float* stage = red_stage_acquire(rs, lane);
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int v = lane + kWarp * q;
        if (v < nv) st_shared4(stage + 4 * v, f4_scale(x[q], nlr_std));
      }
      red_stage_issue(rs, row, dim, lane);
      return;
    }
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int v = lane + kWarp * q;
      if (v < nv) table_red_add4(t, row + 4 * v, f4_scale(x[q], nlr_std));
    }
    return;
  }
  const float stdv = sqrtf(*state_ptr(t, id)) + 1e-10f;
  const float nlr_std = -lr / stdv;               // one division per row: (-lr * g) / std up to one rounding
  for (int v = lane; v < nv; v += kWarp) {
    float4 x = ld4(g + 4 * v);
    table_red_add4(t, row + 4 * v, f4_scale(x, nlr_std));
  }
  for (int k = (nv << 2) + lane; k < dim; k += kWarp) atomicAdd(row + k, (-lr * g[k]) / stdv);
}

__device__ void reduce_log_part(const StepParams& p, const StepWs& w, long long nreg, const float* wbar, float* log4,
                                int bid, int nb);

// Two CTAs per SM (16 warps): the kernel takes 100 registers and spills none.  Held to 64 registers (4 CTAs) it spilled
// its loop state and the bulk-reduction staging state to local memory inside the row loops, and at 80 (3 CTAs) it still
// spilled; on an H100 both were slower (DESIGN.md section 4).
__global__ void __launch_bounds__(kRowBlock, 2) k_update(UpdArgs a) {
  __shared__ __align__(128) float red_stage[kWarpsPerBlock][2][kRedRowFloats];
  const StepParams& p = a.p;
  const StepWs& w = a.w;
  const int lane = threadIdx.x & 31;
  RedStage rs{a.bulk_red ? red_stage[threadIdx.x >> 5][0] : nullptr, 0u};
  RedStage per_lane{nullptr, 0u};
  const int warp0 = (int)blockIdx.x * kWarpsPerBlock + (int)(threadIdx.x >> 5);
  const int nwarps = (int)gridDim.x * kWarpsPerBlock;
  const bool rel_edge = !p.rel_deferred && !p.rel_dense;      // relation entry handled per edge, here
  // phases a.phase_lo..a.phase_hi as straight-line code: a phase counter live across all three cost a spill
  if (a.phase_lo <= 1) {
    const long long nrel = (p.rel_dense && !p.rel_deferred) ? a.rel.num_rows : 0;
    const long long U = node_count(p);
    // a node's id is loaded one job ahead, before the stores of the job in hand: its row loads wait on no index load
    long long id = (warp0 < U) ? a.b.node_ids[warp0] : 0;
    for (long long j = warp0; j < U + nrel; j += nwarps) {
      const long long cur = id;
      if (j + nwarps < U) id = a.b.node_ids[j + nwarps];
      if (j < U) upd_node(p, a.ent, a.b, w, j, cur, lane, rs);
      else upd_rel_dense(a.rel, w.rg, w.rgs, j - U, p.lr, lane);
    }
    if (a.phase_hi > 1) grid_barrier(w.sync_ctr + 0);
  }
  if (a.phase_lo <= 2 && a.phase_hi >= 2) {
    if (p.fused) {
      // mean(G_neg^2) came out of the fused kernel's epilogue: one scalar atomic per negative row
      const long long t0 = (long long)blockIdx.x * blockDim.x + threadIdx.x, nt = (long long)gridDim.x * blockDim.x;
      for (long long j = t0; j < p.Nn; j += nt) table_atomic_add(a.ent, state_ptr(a.ent, a.b.neg_ids[j]), w.gsn[j]);
    } else {
      for (long long j = warp0; j < p.Nn; j += nwarps) {
        const float* g = w.Bn + j * (long long)p.D;
        float gs = 0.f;
        for (int v = lane; v < (p.D >> 2); v += kWarp) { float4 x = ld4(g + 4 * v); gs += f4_dot(x, x); }
        gs = warp_sum(gs);
        if (lane == 0) table_atomic_add(a.ent, state_ptr(a.ent, a.b.neg_ids[j]), gs / (float)p.D);
      }
    }
    if (rel_edge) {
      const long long t0 = (long long)blockIdx.x * blockDim.x + threadIdx.x, nt = (long long)gridDim.x * blockDim.x;
      for (long long i = t0; i < p.B; i += nt) table_atomic_add(a.rel, state_ptr(a.rel, a.b.rel_ids[i]), w.gsr[i]);
    }
    if (a.phase_hi > 2) grid_barrier(w.sync_ctr + 1);
  }
  if (a.phase_hi >= 3) {
    const long long nr = rel_edge ? p.B : 0;
    // the row's index, one job ahead (as in phase 1): the state and gradient loads of a job wait on no index load
    auto job_id = [&](long long j) { return j < p.Nn ? a.b.neg_ids[j] : (j < p.Nn + nr ? a.b.rel_ids[j - p.Nn] : 0); };
    long long id = job_id(warp0);
    for (long long j = warp0; j < p.Nn + nr; j += nwarps) {
      const long long cur = id;
      id = job_id(j + nwarps);
      if (j < p.Nn) apply_row(a.ent, cur, w.Bn + j * (long long)p.D, p.D, p.lr, lane, rs);
      else apply_row(a.rel, cur, w.GR + (j - p.Nn) * (long long)p.Dr, p.Dr, p.lr, lane, per_lane);
    }
    if (a.log4) {
      // on the last CTAs: warps are handed jobs in index order, so those have the fewest rows to apply
      const int nb = gridDim.x < 64 ? gridDim.x : 64;
      const int bid = (int)blockIdx.x - ((int)gridDim.x - nb);
      const bool reg_on = (p.reg_coef > 0.f && p.reg_norm > 0);
      if (bid >= 0)
        reduce_log_part(p, w, reg_on ? (p.B + p.Nn + node_count(p)) : 0, a.wt ? w.wbar : nullptr, a.log4, bid, nb);
    }
  }
  if (rs.buf) red_stage_drain(lane);        // every bulk reduction of this warp has landed
  if (a.phase_hi > a.phase_lo) {
    // leave the barrier counters at zero for the next launch: the last CTA to get here resets them
    __syncthreads();
    if (threadIdx.x == 0) {
      __threadfence();
      if (atomicAdd(w.sync_ctr + 3, 1u) == gridDim.x - 1) {
        w.sync_ctr[0] = 0u; w.sync_ctr[1] = 0u; w.sync_ctr[2] = 0u;
        __threadfence();
        w.sync_ctr[3] = 0u;
      }
    }
  }
}

int launch_update(const LaunchCtx& c, const StepParams& p, const TableView& ent, const TableView& rel,
                  const BatchView& b, const StepWs& w, float* log4, const float* wt) {
  static const bool no_bulk = getenv("KGE_B200_NO_BULKRED") != nullptr;
  UpdArgs a{p, ent, rel, b, w, log4, wt, 1, 3, (!no_bulk && p.D <= kRedRowFloats && (p.D & 3) == 0) ? 1 : 0};
  // job counts per phase (warps): nodes (+ relations), negatives (+ edges), negatives + edges
  const long long nrel = (p.rel_dense && !p.rel_deferred) ? rel.num_rows : 0;
  const long long nr = (!p.rel_deferred && !p.rel_dense) ? p.B : 0;
  long long jobs = p.U + nrel;
  if (p.Nn + nr > jobs) jobs = p.Nn + nr;
  static int occ[64] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev >= 0 && dev < 64 && occ[dev] == 0) {
    int n = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, k_update, kRowBlock, 0) != cudaSuccess || n < 1) n = 1;
    occ[dev] = n;
  }
  static const bool no_coop = getenv("KGE_B200_NO_COOP") != nullptr;
  // multi-GPU: the NCCL all-reduce of the relation sums runs beside this kernel; leave it a few SMs so that the
  // all-or-nothing cooperative launch does not have to wait for it (or it for us)
  const int sms = (p.rel_deferred && c.num_sms > 32) ? c.num_sms - 16 : c.num_sms;
  const int max_resident = sms * (dev >= 0 && dev < 64 ? occ[dev] : 1);
  int grid = ceil_div(jobs, kWarpsPerBlock);
  if (!no_coop) {
    if (grid > max_resident) grid = max_resident;
    void* args[] = {&a};
    prof_begin(c, "k_update<nodes | state adds | apply>");
    cudaError_t e = cudaLaunchCooperativeKernel((void*)k_update, dim3(grid), dim3(kRowBlock), args, 0, c.stream);
    prof_end(c);
    if (c.launch_counter) ++*c.launch_counter;
    if (e == cudaSuccess) return KGE_OK;
    cudaGetLastError();
    return fail(KGE_ERR_CUDA, "cooperative launch of k_update failed: %s (set KGE_B200_NO_COOP=1 for the three-launch form)",
                cudaGetErrorString(e));
  }
  for (int ph = 1; ph <= 3; ++ph) {
    a.phase_lo = a.phase_hi = ph;
    const char* nm = ph == 1 ? "k_update<nodes>" : (ph == 2 ? "k_update<state adds>" : "k_update<apply>");
    KGE_LAUNCH_NAMED(c, nm, k_update, grid, kRowBlock, 0, a);
  }
  return KGE_OK;
}

// one trace entry with possibly duplicated indices (kge_adagrad)
__global__ void __launch_bounds__(kRowBlock) k_state_add(TableView t, const long long* __restrict__ idx,
                                                          const float* __restrict__ grad, long long n, int dim) {
  const long long j = (long long)blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
  if (j >= n) return;
  const int lane = threadIdx.x & 31;
  const float* g = grad + j * (long long)dim;
  float gs = 0.f;
  for (int v = lane; v < (dim >> 2); v += kWarp) { float4 x = ld4(g + 4 * v); gs += f4_dot(x, x); }
  for (int k = ((dim >> 2) << 2) + lane; k < dim; k += kWarp) gs += g[k] * g[k];
  gs = warp_sum(gs);
  if (lane == 0) table_atomic_add(t, state_ptr(t, idx[j]), gs / (float)dim);
}
__global__ void __launch_bounds__(kRowBlock) k_apply(TableView t, const long long* __restrict__ idx,
                                                      const float* __restrict__ grad, long long n, int dim, float lr) {
  const long long j = (long long)blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
  if (j >= n) return;
  RedStage per_lane{nullptr, 0u};
  apply_row(t, idx[j], grad + j * (long long)dim, dim, lr, threadIdx.x & 31, per_lane);
}

// ---- multi-GPU relation path: per-edge gradients -> dense per-relation sums (all-reduced by the host
// with NCCL) -> identical Adagrad on every replica.  Summing the occurrences first is the same math as
// ExternalEmbedding.update: every occurrence is scaled by the same final state (tensor_models.py:352-361).
__global__ void __launch_bounds__(kRowBlock) k_rel_accumulate(StepParams p, BatchView b, StepWs w,
                                                               float* __restrict__ rg, float* __restrict__ rgs) {
  const long long i = (long long)blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
  if (i >= p.B) return;
  const int lane = threadIdx.x & 31;
  const long long rid = b.rel_ids[i];
  const float* g = w.GR + i * (long long)p.Dr;
  float* dst = rg + rid * (long long)p.Dr;
  for (int v = lane; v < (p.Dr >> 2); v += kWarp) red_add4(dst + 4 * v, ld4(g + 4 * v));
  if (lane == 0) atomicAdd(rgs + rid, w.gsr[i]);
}

__global__ void __launch_bounds__(kRowBlock) k_rel_apply_dense(TableView rel, float* __restrict__ rg,
                                                                float* __restrict__ rgs, float lr) {
  const long long r = (long long)blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
  if (r >= rel.num_rows) return;
  const int lane = threadIdx.x & 31;
  const float gs = rgs[r];
  if (gs == 0.f) return;           // relation not touched by any rank this step
  float* st = state_ptr(rel, r);
  float s_new = 0.f;
  if (lane == 0) { s_new = *st + gs; *st = s_new; rgs[r] = 0.f; }
  s_new = __shfl_sync(0xffffffffu, s_new, 0);
  const float stdv = sqrtf(s_new) + 1e-10f;
  float* row = row_ptr(rel, r);
  float* g = rg + r * (long long)rel.dim;
  const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int v = lane; v < (rel.dim >> 2); v += kWarp) {
    float4 x = ld4(g + 4 * v), e = ld4(row + 4 * v);
    st4(row + 4 * v, f4_fma(x, -lr / stdv, e));
    st4(g + 4 * v, z);
  }
}

void launch_rel_grad_dense(const LaunchCtx& c, const StepParams& p, const BatchView& b, const StepWs& w, float* rg,
                           float* rgs) {
  KGE_LAUNCH(c, k_rel_accumulate, ceil_div(p.B, kWarpsPerBlock), kRowBlock, 0, p, b, w, rg, rgs);
}
void launch_rel_apply_dense(const LaunchCtx& c, const TableView& rel, float* rg, float* rgs, float lr) {
  KGE_LAUNCH(c, k_rel_apply_dense, ceil_div(rel.num_rows, kWarpsPerBlock), kRowBlock, 0, rel, rg, rgs, lr);
}

void launch_adagrad(const LaunchCtx& c, const TableView& t, const long long* idx, const float* grad, long long n,
                    float lr) {
  if (n <= 0) return;
  KGE_LAUNCH(c, k_state_add, ceil_div(n, kWarpsPerBlock), kRowBlock, 0, t, idx, grad, n, t.dim);
  KGE_LAUNCH(c, k_apply, ceil_div(n, kWarpsPerBlock), kRowBlock, 0, t, idx, grad, n, t.dim, lr);
}

// debug: out[u,:] = NG[u,:] + reg'(emb[node_ids[u],:])  (what the reference exposes as data.grad)
__global__ void __launch_bounds__(kRowBlock) k_node_grad_reg(StepParams p, TableView ent, BatchView b, StepWs w,
                                                              float* __restrict__ out) {
  const long long u = (long long)blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
  if (u >= node_count(p)) return;
  const int lane = threadIdx.x & 31;
  const float* row = node_row(p, ent, b, w, u);
  for (int v = lane; v < (p.D >> 2); v += kWarp)
    st4(out + u * (long long)p.D + 4 * v,
        f4_add(ld4(w.NG + u * (long long)p.D + 4 * v), reg_grad4(ld4(row + 4 * v), p.reg_norm, p.reg_coef)));
}
void launch_node_grad_with_reg(const LaunchCtx& c, const StepParams& p, const TableView& ent, const BatchView& b,
                               const StepWs& w, float* out) {
  KGE_LAUNCH(c, k_node_grad_reg, ceil_div(p.U, kWarpsPerBlock), kRowBlock, 0, p, ent, b, w, out);
}

}  // namespace kge
