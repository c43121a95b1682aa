// kge_abi.cu -- the extern "C" surface of libkge_b200.so (include/kge_b200.h) and the per-step
// orchestration: which kernels run, in which order, on which workspace.
//
// Step schedule (all on the caller's stream, no host sync):
//   forward_backward:  k_prep -> k_score -> k_loss(+colsum, reduce_log) -> k_grad<A> -> k_grad<B> -> k_chain
//   update:            k_upd_nodes -> k_state_add(negs) -> k_apply(negs) -> k_apply(rels)
// The order of the update kernels reproduces ExternalEmbedding.update's trace-entry order
// (tensor_models.py:316-361, general_models.py:586-588): entity [unique positive nodes, negatives],
// then relation rows; within an entry every state_sum add lands before any row is scaled.
#include <cstdio>
#include <unistd.h>
#include <cstdarg>
#include <cstring>
#include <cstdlib>
#include <map>
#include <mutex>
#include <new>
#include <utility>
#include <cuda.h>
#include "kge_common.cuh"

namespace kge {

namespace {
thread_local char g_err[512] = "";
}  // namespace

int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}

int smem_optin(const void* kernel, size_t bytes) {
  if (bytes <= 48 * 1024) return KGE_OK;
  // umma_supported keeps the shapes that would need more off the wgmma engine
  if (bytes > kSmemOptinMax) return fail(KGE_ERR_UNSUPPORTED, "%zu bytes of shared memory per CTA requested, sm_90 allows %zu", bytes, kSmemOptinMax);
  int dev = 0;
  cudaGetDevice(&dev);
  static std::mutex mu;
  static std::map<std::pair<const void*, int>, size_t> done;
  std::lock_guard<std::mutex> lock(mu);
  size_t& have = done[{kernel, dev}];
  if (bytes <= have) return KGE_OK;
  const cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
  if (e != cudaSuccess) {
    cudaGetLastError();
    return fail(KGE_ERR_CUDA, "cudaFuncSetAttribute(MaxDynamicSharedMemorySize, %zu): %s", bytes, cudaGetErrorString(e));
  }
  have = bytes;
  return KGE_OK;
}

// A buffer the library (re)allocates between steps: device memory, or page-locked host memory (the staging of
// kge_step_fused_host).  The caller decides when and to what size.
struct Buffer {
  void* p = nullptr;
  size_t bytes = 0;
  bool host = false;
  template <class T> T* as() const { return static_cast<T*>(p); }

  void release() {
    if (p) host ? cudaFreeHost(p) : cudaFree(p);
    p = nullptr;
    bytes = 0;
  }
  // Replaces the buffer by one of `n` bytes.  The old one may still be in use by work on `stream`, so this
  // synchronises first, which a stream being captured into a CUDA graph must not do: there it refuses.
  int resize(size_t n, cudaStream_t stream, const char* what) {
    cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
    cudaStreamIsCapturing(stream, &cs);
    if (cs != cudaStreamCaptureStatusNone)
      return fail(KGE_ERR_INVALID_ARG, "the %s must be (re)allocated (%zu bytes, has %zu) but the stream is capturing: "
                  "run one eager step first", what, n, bytes);
    cudaError_t e = cudaStreamSynchronize(stream);
    if (e != cudaSuccess) return fail(KGE_ERR_CUDA, "cudaStreamSynchronize before reallocating the %s: %s", what, cudaGetErrorString(e));
    release();
    e = host ? cudaMallocHost(&p, n) : cudaMalloc(&p, n);
    if (e != cudaSuccess) {
      p = nullptr;
      cudaGetLastError();
      return fail(KGE_ERR_NOMEM, "%s(%zu) for the %s failed: %s", host ? "cudaMallocHost" : "cudaMalloc", n, what,
                  cudaGetErrorString(e));
    }
    bytes = n;
    return KGE_OK;
  }
};

}  // namespace kge
using namespace kge;

#define KGE_CUDA_OK(expr)                                                                      \
  do {                                                                                         \
    cudaError_t e_ = (expr);                                                                   \
    if (e_ != cudaSuccess) return fail(KGE_ERR_CUDA, "%s: %s", #expr, cudaGetErrorString(e_)); \
  } while (0)

struct kge_context {
  int device = 0;
  int num_sms = 0;
  long long launches = 0;
  int engine = -1;
  int rel_deferred = 0;
  // device arena of the step workspace (carve)
  Buffer arena;
  // NG must be zero between steps: remember how much of it has been zeroed
  float* ng_ptr = nullptr;
  size_t ng_floats = 0;
  bool ng_dirty = false;   // a forward_backward whose gradients were never consumed by kge_update
  // pinned + device staging for the *_host entry points
  Buffer pin{nullptr, 0, true};
  Buffer dev_stage;
  float* red_partial = nullptr;      // k_reduce_log partials + ticket + k_update barrier counters (persistent, zero-initialised once)
  Buffer rel_dense;                  // [n_rel * Dr | n_rel] per-relation gradient sums of the fused step (zero between steps)
  float* ext_rg = nullptr;           // deferred relation mode: caller-owned dense buffers [n_rel * Dr], [n_rel] that k_chain sums
  float* ext_rgs = nullptr;          //   the relation gradients into (all-reduced by the caller, kge_set_relation_buffers)
  float* dump_v = nullptr;           // test hook (kge_debug_set_dump): coefficient matrices of the fused kernel
  Buffer negdeg_ids;                 // --neg_deg_sample: the augmented negative id list [C * (Cs + Ns)] of the last step
  Buffer topk_ws;                    // kge_topk: the select CTAs' survivors and the per-list bounds
  Buffer sim_ws;                     // kge_sim_tile: TF32 hi/lo operands and row norms of the GEMM functions
  // kge_set_next_batch: rows of the next step staged by this step's fused kernels
  struct Prefetch {
    bool armed = false;              // a next batch is registered for the coming kge_step_fused_begin
    kge_batch_t next{};
    long long next_nneg = 0;
    bool ready = false;              // the previous begin staged rows for the batch described by r_*
    const void *r_nodes = nullptr, *r_negs = nullptr, *r_nU_dev = nullptr;
    long long r_nU = 0, r_nneg = 0;
    int r_buf = 0;                   // which nc[] holds them
    Buffer nc[2];
    Buffer bn[2];                    // double-buffered like nc: k_fused<N> of step k reads bn[cur] while it stages bn[cur^1]
    FusedPrefetch args{};            // what this step's fused kernels copy

    // `usable`: this step's fused kernels read rows from NC / BnRaw, so staged rows can stand in for its gathers.
    // The rows the previous step staged replace this step's gathers -- only for exactly the batch that was announced.
    void take_staged(const kge_batch_t& b, bool usable, StepParams& p, StepWs& w) {
      if (!ready) return;
      ready = false;
      if (usable && r_nodes == b.node_ids && r_negs == b.neg_ids && r_nU == b.n_nodes &&
          r_nU_dev == (b.n_nodes < 0 ? b.n_nodes_dev : nullptr) && r_nneg == p.Nn) {
        w.NC = nc[r_buf].as<float>();
        w.BnRaw = bn[r_buf].as<float>();
        p.nc_staged = 1;
      }
    }

    // Arms the copy of the announced next batch's rows by this step's fused kernels.  *out: what they copy, or null.
    // `arena_nc`: the workspace's own NC, which this step falls back to when growing the buffers drops the staged rows.
    int arm_next(bool usable, StepParams& p, StepWs& w, float* arena_nc, cudaStream_t stream, const FusedPrefetch** out) {
      *out = nullptr;
      if (!armed) return KGE_OK;
      armed = false;
      const long long ncap = 2 * p.B;
      const long long nU = next.n_nodes < 0 ? ncap : next.n_nodes;
      if (!usable || nU > ncap || next_nneg <= 0 || fused_prefetch_slots(p, 0) < 2 || fused_prefetch_slots(p, 1) < 2)
        return KGE_OK;
      const size_t ncb = (size_t)ncap * p.D * sizeof(float), bnb = (size_t)next_nneg * p.D * sizeof(float);
      if (ncb > nc[0].bytes || ncb > nc[1].bytes || bnb > bn[0].bytes || bnb > bn[1].bytes) {
        for (int i = 0; i < 2; ++i) {
          int rc;
          if ((rc = nc[i].resize(ncb, stream, "prefetch staging buffers")) || (rc = bn[i].resize(bnb, stream, "prefetch staging buffers")))
            return rc;
        }
        w.BnRaw = nullptr; w.NC = arena_nc; p.nc_staged = 0;      // whatever was staged is gone with the old buffers
      }
      const int tgt = p.nc_staged ? (r_buf ^ 1) : 0;
      const void* nU_dev = next.n_nodes < 0 ? next.n_nodes_dev : nullptr;
      args = FusedPrefetch{(const long long*)next.node_ids, (const long long*)nU_dev, nU, (const long long*)next.neg_ids,
                           next_nneg, nc[tgt].as<float>(), bn[tgt].as<float>()};
      ready = true;
      r_nodes = next.node_ids; r_negs = next.neg_ids; r_nU = next.n_nodes; r_nU_dev = nU_dev; r_nneg = next_nneg; r_buf = tgt;
      *out = &args;
      return KGE_OK;
    }
  } pf;
  int fused_mode = -1;               // -1 default (fused kernel whenever the shape allows), 0 off
  float* dev_log4 = nullptr;
  // last step (for kge_update / kge_debug_read)
  StepParams last_p{};
  StepWs last_w{};
  BatchView last_b{};
  TableView last_ent{}, last_rel{};
  bool have_last = false;
  Profiler prof;
};

namespace {

struct DeviceGuard {
  int prev = -1;
  explicit DeviceGuard(int dev) {
    cudaGetDevice(&prev);
    if (prev != dev) cudaSetDevice(dev);
    else prev = -1;
  }
  ~DeviceGuard() {
    if (prev >= 0) cudaSetDevice(prev);
  }
};

int make_view(const kge_table_t* t, TableView* v, const char* what) {
  if (!t || !t->shards) return fail(KGE_ERR_INVALID_ARG, "%s table is null", what);
  if (t->n_shards < 1 || t->n_shards > KGE_MAX_SHARDS)
    return fail(KGE_ERR_INVALID_ARG, "%s table: n_shards=%d out of [1,%d]", what, t->n_shards, KGE_MAX_SHARDS);
  if (t->dim <= 0 || t->num_rows <= 0) return fail(KGE_ERR_INVALID_ARG, "%s table: empty", what);
  memset(v, 0, sizeof(*v));
  v->n_shards = t->n_shards;
  v->dim = t->dim;
  v->num_rows = t->num_rows;
  v->rows_per_shard = (t->num_rows + t->n_shards - 1) / t->n_shards;
  for (int s = 0; s < t->n_shards; ++s) {
    const kge_shard_t& sh = t->shards[s];
    long long begin = (long long)s * v->rows_per_shard;
    long long end = begin + v->rows_per_shard;
    if (end > t->num_rows) end = t->num_rows;
    if (sh.row_begin != begin || sh.row_end != end || sh.dim != t->dim)
      return fail(KGE_ERR_INVALID_ARG, "%s table: shard %d must cover rows [%lld,%lld) with dim %d", what, s, begin,
                  end, t->dim);
    if (!sh.emb || !sh.state_sum) return fail(KGE_ERR_INVALID_ARG, "%s table: shard %d has null pointers", what, s);
    if (((uintptr_t)sh.emb & 15) != 0) return fail(KGE_ERR_INVALID_ARG, "%s table: shard %d not 16-byte aligned", what, s);
    v->emb[s] = sh.emb;
    v->state[s] = sh.state_sum;
  }
  return KGE_OK;
}

int make_params(const kge_step_cfg_t* cfg, long long n_nodes, StepParams* p) {
  if (!cfg) return fail(KGE_ERR_INVALID_ARG, "cfg is null");
  if (cfg->model < KGE_TRANSE_L1 || cfg->model > KGE_ROTATE) return fail(KGE_ERR_INVALID_ARG, "unknown model %d", cfg->model);
  if (cfg->batch <= 0 || cfg->chunk_size <= 0 || cfg->neg_sample_size <= 0)
    return fail(KGE_ERR_INVALID_ARG, "batch/chunk_size/neg_sample_size must be positive");
  // the reference skips ragged batches (dataloader/sampler.py:503-504)
  if (cfg->batch % cfg->chunk_size != 0)
    return fail(KGE_ERR_INVALID_ARG, "batch %lld is not a multiple of chunk_size %d", (long long)cfg->batch, cfg->chunk_size);
  const int D = cfg->entity_dim, Dr = cfg->relation_dim;
  if (D <= 0 || Dr <= 0) return fail(KGE_ERR_INVALID_ARG, "dims must be positive");
  if (D % 4 != 0 || Dr % 4 != 0)
    return fail(KGE_ERR_UNSUPPORTED, "row lengths must be multiples of 4 floats (16-byte vector/TMA access): D_e=%d D_r=%d", D, Dr);
  switch (cfg->model) {
    case KGE_TRANSE_L1: case KGE_TRANSE_L2: case KGE_DISTMULT:
      if (Dr != D) return fail(KGE_ERR_INVALID_ARG, "model needs relation_dim == entity_dim (%d vs %d)", Dr, D);
      break;
    case KGE_COMPLEX:
      if (Dr != D || D % 8 != 0) return fail(KGE_ERR_INVALID_ARG, "ComplEx needs relation_dim == entity_dim, a multiple of 8");
      break;
    case KGE_ROTATE:
      if (D != 2 * Dr || D % 8 != 0) return fail(KGE_ERR_INVALID_ARG, "RotatE needs entity_dim == 2*relation_dim (-de), a multiple of 8");
      break;
    case KGE_RESCAL:
      if (Dr != D * D) return fail(KGE_ERR_INVALID_ARG, "RESCAL needs relation_dim == entity_dim^2");
      if (D > 512) return fail(KGE_ERR_UNSUPPORTED, "RESCAL entity_dim %d > 512 is not implemented", D);
      break;
  }
  p->model = cfg->model; p->D = D; p->Dr = Dr;
  p->gamma = cfg->gamma; p->emb_init = cfg->emb_init; p->lr = cfg->lr;
  p->reg_coef = cfg->reg_coef; p->reg_norm = cfg->reg_norm;
  p->adversarial = cfg->adversarial; p->adv_temperature = cfg->adv_temperature;
  p->neg_head = cfg->neg_head ? 1 : 0;
  p->B = cfg->batch; p->Cs = cfg->chunk_size; p->Ns = cfg->neg_sample_size;
  p->C = (int)(cfg->batch / cfg->chunk_size);
  // --neg_deg_sample: every chunk's negatives are its own Cs corrupted-side rows followed by the Ns sampled ones
  p->neg_deg = cfg->neg_deg_sample ? 1 : 0;
  if (p->neg_deg) p->Ns += p->Cs;
  p->Nn = (long long)p->C * p->Ns;
  p->U = n_nodes >= 0 ? n_nodes : 2 * p->B;      // capacity when only the device knows the count
  p->U_dev = nullptr;
  p->rel_deferred = 0; p->rel_dense = 0; p->use_nc = 1; p->fused = 0; p->nc_staged = 0;
  if (cfg->loss_genre < KGE_LOSS_LOGSIGMOID || cfg->loss_genre > KGE_LOSS_BCE)
    return fail(KGE_ERR_INVALID_ARG, "loss_genre %d is not a kge_loss_t", cfg->loss_genre);
  if (cfg->pairwise && cfg->loss_genre != KGE_LOSS_HINGE && cfg->loss_genre != KGE_LOSS_LOGISTIC)
    return fail(KGE_ERR_INVALID_ARG, "pairwise needs the Hinge or the Logistic criterion (loss.py:61-62)");
  if (cfg->pairwise && cfg->adversarial)
    return fail(KGE_ERR_INVALID_ARG, "loss cannot be pairwise and adversarial sampled (base_loss.py:83-84)");
  p->hinge = cfg->loss_genre == KGE_LOSS_HINGE ? 1 : 0;
  p->margin = cfg->margin;
  p->pairwise = cfg->pairwise ? 1 : 0;
  return KGE_OK;
}

size_t align_up(size_t x, size_t a = 256) { return (x + a - 1) / a * a; }

// Carves the step workspace out of the arena; grows the arena if needed.
// Layout rule: every buffer whose size depends only on (B, Ns, D) comes first, the buffers that depend on the unique-node
// count U (NC, regp) come last -- the TMA tensor maps of the GEMM operands are cached by base address, and U changes
// every step.
struct CarveOpt {
  bool force_tiles = false;   // fp32 CUDA-core tiles regardless of the handle's engine (kge_score_neg for RESCAL)
  bool want_scores = true;    // fused path: keep a [B, Ns] score matrix for kge_debug_read
};

bool use_fused(kge_context* h, const StepParams& p) {
  return h->engine != 0 && h->fused_mode != 0 && fused_supported(p);
}

bool use_umma(kge_context* h, const StepParams& p) {
  return h->engine != 0 && umma_supported(p);    // engine -1 (default) / 1: wgmma whenever the shape allows it
}

int carve(kge_context* h, const StepParams& p, StepWs* w, cudaStream_t stream, const CarveOpt& opt = CarveOpt()) {
  const size_t BD = (size_t)p.B * p.D, ND = (size_t)p.Nn * p.D, BNs = (size_t)p.B * p.Ns;
  const size_t B = (size_t)p.B, Nn = (size_t)p.Nn, U = (size_t)(p.U > 0 ? p.U : 0);
  const bool um = !opt.force_tiles && use_umma(h, p);
  const bool fused = p.fused != 0;
  const FusedHilo hl = fused ? fused_hilo(p) : FusedHilo{false, false};
  // slab layout pads the blocked dimension to a multiple of 32 (+ one slab of slack for box overruns)
  const size_t sA = B * slab_blocks(p.D) * 32 + 8192, sB = Nn * slab_blocks(p.D) * 32 + 8192;
  const size_t sV = B * slab_blocks(p.Ns) * 32 + 8192;
  // transposed slabs: [C][rows / 32][cols][32]
  const size_t sAT = (size_t)p.C * slab_blocks(p.Cs) * p.D * 32 + 8192, sBT = (size_t)p.C * slab_blocks(p.Ns) * p.D * 32 + 8192;
  const size_t sVT = (size_t)p.C * slab_blocks(p.Cs) * p.Ns * 32 + 8192;
  struct Slot { float** ptr; size_t floats; bool on; };
  const Slot slots[] = {
      // NG first, sized for the largest possible node count (2B): rows >= U are never written, rows < U are
      // re-zeroed by the node update, so one fill keeps the whole region zero across steps with varying U
      {&w->NG, (U ? 2 * B : 0) * p.D, true},
      {&w->A, BD, !(um || fused)}, {&w->Bn, ND, true}, {&w->GA, BD, true}, {&w->GR, B * p.Dr, !p.rel_dense},
      {&w->S, BNs, !fused || opt.want_scores}, {&w->V, BNs, !fused},
      {&w->pos, B, true}, {&w->gpos, B, true}, {&w->pnorm, B, true}, {&w->a2, B, true}, {&w->b2, Nn, true},
      {&w->rowsum, B, true}, {&w->colsum, Nn, true}, {&w->pl, B, true}, {&w->nl, B, true}, {&w->wbar, 4, true},
      {&w->gsr, B, true}, {&w->gsn, Nn, true}, {&w->colpart, (size_t)ceil_div(p.Cs, 128) * Nn, fused},
      {&w->Mt, BD, p.model == KGE_RESCAL},
      {&w->Ahi, sA, um && (!fused || hl.a)}, {&w->Alo, sA, um && (!fused || hl.a)}, {&w->Af, sA, fused && !hl.a},
      {&w->Bhi, sB, um}, {&w->Blo, sB, um},
      {&w->Vhi, sV, um && !fused}, {&w->Vlo, sV, um && !fused},
      {&w->AhiT, sAT, um}, {&w->AloT, sAT, um}, {&w->BhiT, sBT, um}, {&w->BloT, sBT, um},
      {&w->VhiT, sVT, um && (!fused || hl.v)}, {&w->VloT, sVT, um && (!fused || hl.v)}, {&w->VT, sVT, fused},
      // U-dependent tail
      {&w->NC, U * p.D, p.use_nc != 0},
      {&w->regp, B + Nn + (U ? 2 * B : 0), true},
  };
  size_t need = 0;
  for (const Slot& s : slots)
    if (s.on) need += align_up(s.floats * sizeof(float));
  if (need > h->arena.bytes) {
    if (int rc = h->arena.resize(need + need / 4, stream, "step workspace")) return rc;
    h->ng_ptr = nullptr; h->ng_floats = 0;
  }
  size_t off = 0;
  for (const Slot& s : slots) {
    *s.ptr = s.on ? (float*)(h->arena.as<char>() + off) : nullptr;
    if (s.on) off += align_up(s.floats * sizeof(float));
  }
  w->red_partial = h->red_partial; w->red_ticket = (unsigned int*)(h->red_partial + 192);
  w->sync_ctr = (unsigned int*)(h->red_partial + 200);
  w->rg = nullptr; w->rgs = nullptr;
  return KGE_OK;
}

// dense per-relation gradient buffers of the fused single-GPU step (zero between steps: the update re-zeroes what it consumes)
int ensure_rel_dense(kge_context* h, const TableView& rel, StepWs* w, cudaStream_t stream) {
  const size_t bytes = ((size_t)rel.num_rows * rel.dim + (size_t)rel.num_rows) * sizeof(float);
  if (bytes != h->rel_dense.bytes) {
    if (int rc = h->rel_dense.resize(bytes, stream, "relation gradient sums")) return rc;
    KGE_CUDA_OK(cudaMemsetAsync(h->rel_dense.p, 0, bytes, stream));
  }
  w->rg = h->rel_dense.as<float>();
  w->rgs = w->rg + (size_t)rel.num_rows * rel.dim;
  return KGE_OK;
}

LaunchCtx lctx(kge_context* h, void* stream) { return LaunchCtx{(cudaStream_t)stream, &h->launches, h->num_sms, &h->prof}; }

// NG (node-gradient accumulator) has to be zero when k_chain starts.  k_upd_nodes re-zeroes the
// rows it consumes, so only a fresh / enlarged region needs an explicit fill.
void ensure_ng_zero(kge_context* h, const StepParams& p, const StepWs& w, const LaunchCtx& c, bool force) {
  size_t n = (size_t)2 * p.B * p.D;
  if (force || h->ng_dirty || h->ng_ptr != w.NG || h->ng_floats < n) {
    launch_fill_zero(c, w.NG, (long long)n);
    h->ng_ptr = w.NG;
    h->ng_dirty = false;
  }
  h->ng_floats = n;   // only [0, n) is guaranteed zero after this step (the region beyond is reused)
}

int check_batch(const kge_batch_t* b, const StepParams& p) {
  if (!b) return fail(KGE_ERR_INVALID_ARG, "batch is null");
  if (!b->node_ids || !b->head_local || !b->tail_local || !b->rel_ids || !b->neg_ids)
    return fail(KGE_ERR_INVALID_ARG, "batch has null index arrays");
  if (b->n_nodes < 0 && b->n_nodes_dev) return KGE_OK;      // device-side count (kge_sampler_sample)
  if (b->n_nodes <= 0 || b->n_nodes > 2 * p.B) return fail(KGE_ERR_INVALID_ARG, "n_nodes=%lld out of (0, 2*batch]", (long long)b->n_nodes);
  return KGE_OK;
}

BatchView bview(const kge_batch_t* b) {
  return BatchView{(const long long*)b->node_ids, (const long long*)b->head_local, (const long long*)b->tail_local,
                   (const long long*)b->rel_ids, (const long long*)b->neg_ids, b->edge_weight,
                   (const long long*)b->head_ids, (const long long*)b->tail_ids};
}

int run_score(kge_context* h, const LaunchCtx& c, const StepParams& p, const StepWs& w) {
  if (use_umma(h, p)) return umma_score(c, p, w);
  launch_score(c, p, w);
  return KGE_OK;
}

}  // namespace

extern "C" {

KGE_API int kge_abi_version(void) { return KGE_ABI_VERSION; }
KGE_API const char* kge_last_error(void) { return g_err; }

KGE_API int kge_create(int device, kge_handle_t* out) {
  if (!out) return fail(KGE_ERR_INVALID_ARG, "out is null");
  *out = nullptr;
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n == 0) {
    cudaGetLastError();
    return fail(KGE_ERR_NO_DEVICE, "no CUDA device visible (%s); libkge_b200 has no CPU path", cudaGetErrorString(e));
  }
  if (device < 0 || device >= n) return fail(KGE_ERR_INVALID_ARG, "device %d out of range [0,%d)", device, n);
  cudaDeviceProp prop;
  KGE_CUDA_OK(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9)
    return fail(KGE_ERR_NO_DEVICE, "device %d is sm_%d%d; this library is built for sm_90a (H100) only", device, prop.major, prop.minor);
  kge_context* h = new (std::nothrow) kge_context();
  if (!h) return fail(KGE_ERR_NOMEM, "out of host memory");
  h->device = device;
  h->num_sms = prop.multiProcessorCount;
  if (const char* ev = getenv("KGE_B200_FUSED")) h->fused_mode = atoi(ev) ? 1 : 0;   // A/B switch for benchmarks

  DeviceGuard g(device);
  if (cudaMalloc(&h->dev_log4, 4 * sizeof(float)) != cudaSuccess) { delete h; return fail(KGE_ERR_NOMEM, "cudaMalloc failed"); }

  if (cudaMalloc(&h->red_partial, 256 * sizeof(float)) != cudaSuccess || cudaMemset(h->red_partial, 0, 256 * sizeof(float)) != cudaSuccess) {
    delete h; return fail(KGE_ERR_NOMEM, "cudaMalloc failed");
  }
  *out = h;
  return KGE_OK;
}

KGE_API int kge_destroy(kge_handle_t h) {
  if (!h) return KGE_OK;
  DeviceGuard g(h->device);
  cudaDeviceSynchronize();
  for (Buffer* b : {&h->arena, &h->dev_stage, &h->pin, &h->rel_dense, &h->negdeg_ids, &h->topk_ws, &h->sim_ws, &h->pf.nc[0], &h->pf.nc[1],
                    &h->pf.bn[0], &h->pf.bn[1]})
    b->release();
  if (h->dev_log4) cudaFree(h->dev_log4);
  if (h->red_partial) cudaFree(h->red_partial);
  if (h->prof.created)
    for (int i = 0; i < Profiler::kMax; ++i) { cudaEventDestroy(h->prof.ev0[i]); cudaEventDestroy(h->prof.ev1[i]); }
  delete h;
  return KGE_OK;
}

KGE_API int64_t kge_launch_count(kge_handle_t h) { return h ? h->launches : 0; }

KGE_API int kge_profile_enable(kge_handle_t h, int on) {
  if (!h) return fail(KGE_ERR_INVALID_ARG, "handle is null");
  DeviceGuard g(h->device);
  Profiler& p = h->prof;
  if (on && !p.created) {
    for (int i = 0; i < Profiler::kMax; ++i) {
      KGE_CUDA_OK(cudaEventCreate(&p.ev0[i]));
      KGE_CUDA_OK(cudaEventCreate(&p.ev1[i]));
    }
    p.created = true;
  }
  p.enabled = on != 0;
  p.n = 0;
  return KGE_OK;
}

KGE_API int kge_profile_read(kge_handle_t h, char* names, int names_len, float* ms, int max_records) {
  if (!h || !names || !ms) return fail(KGE_ERR_INVALID_ARG, "null argument");
  DeviceGuard g(h->device);
  Profiler& p = h->prof;
  KGE_CUDA_OK(cudaDeviceSynchronize());
  int n = p.n < max_records ? p.n : max_records, off = 0;
  names[0] = 0;
  for (int i = 0; i < n; ++i) {
    KGE_CUDA_OK(cudaEventElapsedTime(&ms[i], p.ev0[i], p.ev1[i]));
    int w = snprintf(names + off, names_len - off, "%s%s", i ? "|" : "", p.names[i]);
    if (w < 0 || off + w >= names_len) break;
    off += w;
  }
  p.n = 0;   // start a new record set
  return n;
}

KGE_API int kge_set_engine(kge_handle_t h, int engine) {
  if (!h) return fail(KGE_ERR_INVALID_ARG, "handle is null");
  if (engine < -1 || engine > 1) return fail(KGE_ERR_INVALID_ARG, "engine must be -1, 0 or 1");
  h->engine = engine;
  return KGE_OK;
}

KGE_API int kge_set_fused(kge_handle_t h, int mode) {
  if (!h) return fail(KGE_ERR_INVALID_ARG, "handle is null");
  if (mode < -1 || mode > 1) return fail(KGE_ERR_INVALID_ARG, "mode must be -1, 0 or 1");
  h->fused_mode = mode;
  return KGE_OK;
}

KGE_API int kge_debug_set_dump(kge_handle_t h, float* coef_dump) {
  if (!h) return fail(KGE_ERR_INVALID_ARG, "handle is null");
  h->dump_v = coef_dump;
  return KGE_OK;
}

KGE_API int kge_gather(kge_handle_t h, const kge_table_t* table, const int64_t* idx, int64_t n, float* out, void* stream) {
  if (!h) return fail(KGE_ERR_INVALID_ARG, "handle is null");
  if (n < 0) return fail(KGE_ERR_INVALID_ARG, "n < 0");
  if (n == 0) return KGE_OK;
  if (!idx || !out) return fail(KGE_ERR_INVALID_ARG, "idx/out is null");
  TableView v;
  int rc = make_view(table, &v, "gather");
  if (rc) return rc;
  DeviceGuard g(h->device);
  launch_gather(lctx(h, stream), v, (const long long*)idx, n, out);
  KGE_CUDA_OK(cudaGetLastError());
  return KGE_OK;
}

KGE_API int kge_score_pos(kge_handle_t h, const kge_step_cfg_t* cfg, const float* head, const float* rel, const float* tail,
                  int64_t n, float* out, void* stream) {
  if (!h) return fail(KGE_ERR_INVALID_ARG, "handle is null");
  if (!cfg) return fail(KGE_ERR_INVALID_ARG, "cfg is null");
  if (n == 0) return KGE_OK;
  if (!head || !rel || !tail || !out || n < 0) return fail(KGE_ERR_INVALID_ARG, "bad arguments");
  kge_step_cfg_t c2 = *cfg;
  c2.batch = n; c2.chunk_size = (int32_t)1; c2.neg_sample_size = 1;
  if (n > 0x7fffffffLL) return fail(KGE_ERR_INVALID_ARG, "n too large");
  StepParams p;
  int rc = make_params(&c2, 0, &p);
  if (rc) return rc;
  DeviceGuard g(h->device);
  StepWs w{};
  w.pos = out;
  LaunchCtx c = lctx(h, stream);
  if (p.model == KGE_RESCAL) launch_rescal_prep_dense(c, p, head, rel, tail, w, true, false);
  else launch_prep_dense(c, p, head, rel, tail, nullptr, w, true, false);
  KGE_CUDA_OK(cudaGetLastError());
  return KGE_OK;
}

KGE_API int kge_score_neg(kge_handle_t h, const kge_step_cfg_t* cfg, const float* heads, const float* rel, const float* tails,
                  float* out, void* stream) {
  if (!h) return fail(KGE_ERR_INVALID_ARG, "handle is null");
  if (!heads || !rel || !tails || !out) return fail(KGE_ERR_INVALID_ARG, "null pointer");
  StepParams p;
  int rc = make_params(cfg, 0, &p);
  if (rc) return rc;
  DeviceGuard g(h->device);
  StepWs w{};
  // RESCAL: the a-side kernel (M_r . p) does not split the dense negative rows for the tensor-core engine; its
  // stand-alone negative score runs on the fp32 tile kernels
  CarveOpt opt;
  opt.force_tiles = (p.model == KGE_RESCAL);
  rc = carve(h, p, &w, (cudaStream_t)stream, opt);
  if (rc) return rc;
  h->ng_ptr = nullptr;      // this carve overlays the node-gradient region
  LaunchCtx c = lctx(h, stream);
  // positives' entity rows / negative rows by corruption mode (general_models.py:405-406, 426-427)
  const float* negrows = p.neg_head ? heads : tails;
  if (p.model == KGE_RESCAL) launch_rescal_prep_dense(c, p, heads, rel, tails, w, false, true);
  else launch_prep_dense(c, p, heads, rel, tails, negrows, w, false, true);
  // the tile kernels read the negatives from w.Bn; point it at the caller's rows (read-only here)
  StepWs w2 = w;
  w2.Bn = const_cast<float*>(negrows);
  w2.S = out;
  if (opt.force_tiles) launch_score(c, p, w2);
  else rc = run_score(h, c, p, w2);
  if (rc) return rc;
  KGE_CUDA_OK(cudaGetLastError());
  h->have_last = false;
  return KGE_OK;
}

KGE_API int kge_rank_count(kge_handle_t h, const float* S, int64_t ld, int64_t Q, int64_t N, const float* pos,
                           int64_t base, const int64_t* cand, int64_t chunk, const int64_t* kept, const int64_t* rel,
                           const kge_filter_t* filter, int64_t* cnt, void* stream) {
  if (!h) return fail(KGE_ERR_INVALID_ARG, "handle is null");
  if (Q < 0 || N < 0 || ld < N) return fail(KGE_ERR_INVALID_ARG, "bad tile shape Q=%lld N=%lld ld=%lld", (long long)Q,
                                            (long long)N, (long long)ld);
  if (Q == 0 || N == 0) return KGE_OK;
  if (!S || !pos || !cnt) return fail(KGE_ERR_INVALID_ARG, "null pointer");
  if (cand && chunk <= 0) return fail(KGE_ERR_INVALID_ARG, "chunk must be positive with explicit candidates");
  if (!cand && base < 0) return fail(KGE_ERR_INVALID_ARG, "base < 0");
  const bool filt = filter && filter->n_keys > 0;
  if (filt && (!filter->keys || !filter->vals || !kept || !rel || filter->n_rel <= 0))
    return fail(KGE_ERR_INVALID_ARG, "filter needs keys, vals, kept, rel and n_rel > 0");
  if (Q * ((N + 1023) / 1024) > 0x7fffffffLL) return fail(KGE_ERR_INVALID_ARG, "tile too large");
  RankParams p{};
  p.S = S; p.ld = ld; p.Q = Q; p.N = N; p.pos = pos;
  p.base = base; p.cand = (const long long*)cand; p.chunk = chunk;
  p.kept = (const long long*)kept; p.rel = (const long long*)rel;
  p.keys = filt ? (const long long*)filter->keys : nullptr;
  p.vals = filt ? (const int*)filter->vals : nullptr;
  p.n_keys = filt ? filter->n_keys : 0;
  p.n_rel = filt ? filter->n_rel : 1;
  p.cnt = (long long*)cnt;
  DeviceGuard g(h->device);
  launch_rank_count(lctx(h, stream), p);
  KGE_CUDA_OK(cudaGetLastError());
  return KGE_OK;
}

KGE_API int kge_rank_finish(kge_handle_t h, const int64_t* cnt, int64_t Q, int64_t* rank_out, double* acc, void* stream) {
  if (!h) return fail(KGE_ERR_INVALID_ARG, "handle is null");
  if (Q < 0) return fail(KGE_ERR_INVALID_ARG, "Q < 0");
  if (Q == 0) return KGE_OK;
  if (!cnt || !acc) return fail(KGE_ERR_INVALID_ARG, "null pointer");
  DeviceGuard g(h->device);
  launch_rank_finish(lctx(h, stream), (const long long*)cnt, Q, (long long*)rank_out, acc);
  KGE_CUDA_OK(cudaGetLastError());
  return KGE_OK;
}

KGE_API int kge_topk(kge_handle_t h, const float* S, int64_t ld, int64_t Q, int64_t N, const int64_t* qgroup,
                     const int64_t* qoff, int64_t cbase, int64_t cstride, int32_t K, int64_t G, float* top_score,
                     int64_t* top_key, void* stream) {
  if (!h) return fail(KGE_ERR_INVALID_ARG, "handle is null");
  if (K > KGE_TOPK_MAX) return fail(KGE_ERR_UNSUPPORTED, "K=%d: kge_topk keeps at most KGE_TOPK_MAX=%d entries per list",
                                    (int)K, KGE_TOPK_MAX);
  if (K < 1) return fail(KGE_ERR_INVALID_ARG, "K=%d must be positive", (int)K);
  if (Q < 0 || N < 0 || ld < N || G < 1) return fail(KGE_ERR_INVALID_ARG, "bad tile shape Q=%lld N=%lld ld=%lld G=%lld",
                                                    (long long)Q, (long long)N, (long long)ld, (long long)G);
  if (cbase < 0 || cstride < 1) return fail(KGE_ERR_INVALID_ARG, "cbase=%lld must be >= 0 and cstride=%lld >= 1",
                                            (long long)cbase, (long long)cstride);
  if (Q == 0 || N == 0) return KGE_OK;
  if (!S || !qgroup || !qoff || !top_score || !top_key) return fail(KGE_ERR_INVALID_ARG, "null pointer");
  if (Q * ((N + kTopkSeg - 1) / kTopkSeg) > 0x7fffffffLL || Q > 0x7fffffffLL) return fail(KGE_ERR_INVALID_ARG, "tile too large");
  DeviceGuard g(h->device);
  const cudaStream_t st = (cudaStream_t)stream;
  const size_t bytes = topk_workspace_bytes(Q, N, K, G);
  if (h->topk_ws.bytes < bytes) {
    const int rc = h->topk_ws.resize(bytes, st, "top-K workspace");
    if (rc) return rc;
  }
  TopkParams p{};
  p.S = S; p.ld = ld; p.Q = Q; p.N = N;
  p.qgroup = (const long long*)qgroup; p.qoff = (const long long*)qoff;
  p.cbase = cbase; p.cstride = cstride; p.K = K;
  p.top_score = top_score; p.top_key = (long long*)top_key;
  topk_carve(p, h->topk_ws.p);
  KGE_CUDA_OK(cudaMemsetAsync(p.bound, 0, (size_t)G * sizeof(unsigned), st));
  launch_topk(lctx(h, stream), p);
  KGE_CUDA_OK(cudaGetLastError());
  return KGE_OK;
}

namespace {
int check_sim_args(kge_handle_t h, int32_t sim, const float* left, const float* right, int32_t dim, const float* out) {
  if (!h) return fail(KGE_ERR_INVALID_ARG, "handle is null");
  if (sim < KGE_SIM_COSINE || sim > KGE_SIM_EXT_JACCARD) return fail(KGE_ERR_INVALID_ARG, "unknown similarity %d", (int)sim);
  if (dim < 1 || dim > 160000) return fail(KGE_ERR_UNSUPPORTED, "dim=%d: kge_sim takes 1 <= dim <= 160000", (int)dim);
  if (!left || !right || !out) return fail(KGE_ERR_INVALID_ARG, "null pointer");
  return KGE_OK;
}
}  // namespace

KGE_API int kge_sim_tile(kge_handle_t h, int32_t sim, const float* left, int64_t nL, const float* right, int64_t nR,
                         int32_t dim, float* out, void* stream) {
  if (nL < 0 || nR < 0) return fail(KGE_ERR_INVALID_ARG, "bad tile shape nL=%lld nR=%lld", (long long)nL, (long long)nR);
  if (nL == 0 || nR == 0) return h ? KGE_OK : fail(KGE_ERR_INVALID_ARG, "handle is null");
  if (int rc = check_sim_args(h, sim, left, right, dim, out)) return rc;
  // grid rows (left tiles of 64) and columns (right tiles of 256) stay within the launch limits, and the TMA row
  // coordinate of a slab, (32-column block) * n + row, within int32
  const long long nblk = (dim + 31) / 32;
  if (nL > 65535LL * 64 || nR > 65535LL * 256 || nblk * nL > 0x7fffffffLL || nblk * nR > 0x7fffffffLL)
    return fail(KGE_ERR_INVALID_ARG, "tile too large: nL=%lld nR=%lld dim=%d", (long long)nL, (long long)nR, (int)dim);
  DeviceGuard g(h->device);
  const cudaStream_t st = (cudaStream_t)stream;
  if (sim_uses_gemm(sim)) {
    const size_t bytes = sim_workspace_bytes(nL, nR, dim);
    if (h->sim_ws.bytes < bytes) {
      const int rc = h->sim_ws.resize(bytes, st, "similarity workspace");
      if (rc) return rc;
    }
  }
  if (int rc = launch_sim_tile(lctx(h, stream), sim, left, nL, right, nR, dim, out, h->sim_ws.p)) return rc;
  KGE_CUDA_OK(cudaGetLastError());
  return KGE_OK;
}

KGE_API int kge_sim_pairs(kge_handle_t h, int32_t sim, const float* left, const float* right, int64_t n, int32_t dim,
                          float* out, void* stream) {
  if (n < 0) return fail(KGE_ERR_INVALID_ARG, "n=%lld < 0", (long long)n);
  if (n == 0) return h ? KGE_OK : fail(KGE_ERR_INVALID_ARG, "handle is null");
  if (int rc = check_sim_args(h, sim, left, right, dim, out)) return rc;
  if ((n + 7) / 8 > 0x7fffffffLL) return fail(KGE_ERR_INVALID_ARG, "too many pairs: %lld", (long long)n);
  DeviceGuard g(h->device);
  launch_sim_pairs(lctx(h, stream), sim, left, right, n, dim, out);
  KGE_CUDA_OK(cudaGetLastError());
  return KGE_OK;
}

KGE_API int kge_loss_grad(kge_handle_t h, const kge_step_cfg_t* cfg, const float* pos, const float* neg, const float* wt,
                  float* dpos, float* dneg, float* log4, void* stream) {
  if (!h) return fail(KGE_ERR_INVALID_ARG, "handle is null");
  if (!pos || !neg || !dpos || !dneg) return fail(KGE_ERR_INVALID_ARG, "null pointer");
  StepParams p;
  int rc = make_params(cfg, 0, &p);
  if (rc) return rc;
  p.model = KGE_DISTMULT;   // plain d loss / d score (no distance folding)
  DeviceGuard g(h->device);
  StepWs w{};
  rc = carve(h, p, &w, (cudaStream_t)stream);
  if (rc) return rc;
  h->ng_ptr = nullptr;      // this carve overlays the node-gradient region
  w.V = dneg;
  w.gpos = dpos;
  launch_loss(lctx(h, stream), p, pos, neg, wt, w, log4, false);
  KGE_CUDA_OK(cudaGetLastError());
  h->have_last = false;
  return KGE_OK;
}

KGE_API int kge_adagrad(kge_handle_t h, const kge_table_t* table, const int64_t* idx, const float* grad, int64_t n, float lr,
                void* stream) {
  if (!h) return fail(KGE_ERR_INVALID_ARG, "handle is null");
  if (n < 0) return fail(KGE_ERR_INVALID_ARG, "n < 0");
  if (n == 0) return KGE_OK;
  if (!idx || !grad) return fail(KGE_ERR_INVALID_ARG, "null pointer");
  TableView v;
  int rc = make_view(table, &v, "adagrad");
  if (rc) return rc;
  DeviceGuard g(h->device);
  launch_adagrad(lctx(h, stream), v, (const long long*)idx, grad, n, lr);
  KGE_CUDA_OK(cudaGetLastError());
  return KGE_OK;
}

// One step's forward + backward.  `fused_step`: called from kge_step_fused (nobody reads per-edge relation gradients or
// the score matrix; head/tail rows may be read straight from the table; the log scalars are reduced by the update).
static int forward_backward_impl(kge_handle_t h, const kge_step_cfg_t* cfg, const kge_table_t* ent, const kge_table_t* rel,
                                 const kge_batch_t* batch, float* log4, void* stream, bool fused_step) {
  if (!h) return fail(KGE_ERR_INVALID_ARG, "handle is null");
  StepParams p;
  int rc = make_params(cfg, batch ? batch->n_nodes : 0, &p);
  if (rc) return rc;
  rc = check_batch(batch, p);
  if (rc) return rc;
  if (batch->n_nodes < 0) p.U_dev = (const long long*)batch->n_nodes_dev;
  p.rel_deferred = h->rel_deferred;
  TableView ve, vr;
  if ((rc = make_view(ent, &ve, "entity"))) return rc;
  if ((rc = make_view(rel, &vr, "relation"))) return rc;
  if (ve.dim != p.D || vr.dim != p.Dr)
    return fail(KGE_ERR_INVALID_ARG, "table dims (%d,%d) do not match cfg (%d,%d)", ve.dim, vr.dim, p.D, p.Dr);
  DeviceGuard g(h->device);
  p.fused = use_fused(h, p) ? 1 : 0;
  // fused step on one GPU: nothing can change a table row between its gather and the node update, so the gathered
  // copy NC is skipped; relation gradients are summed per relation (<= 256 MB of sums) instead of stored per edge
  p.use_nc = (fused_step && ve.n_shards == 1) ? 0 : 1;
  p.rel_dense = (fused_step && p.model != KGE_RESCAL &&
                 (p.rel_deferred ? (h->ext_rg != nullptr) : ((size_t)vr.num_rows * (size_t)vr.dim <= ((size_t)64 << 20)))) ? 1 : 0;
  StepWs w{};
  CarveOpt opt;
  opt.want_scores = !fused_step;
  if ((rc = carve(h, p, &w, (cudaStream_t)stream, opt))) return rc;
  if (p.rel_dense && p.rel_deferred) { w.rg = h->ext_rg; w.rgs = h->ext_rgs; }
  else if (p.rel_dense && (rc = ensure_rel_dense(h, vr, &w, (cudaStream_t)stream))) return rc;
  LaunchCtx c = lctx(h, stream);
  BatchView b = bview(batch);
  if (p.neg_deg) {
    if (ve.n_shards != 1) return fail(KGE_ERR_UNSUPPORTED, "--neg_deg_sample needs a single-shard entity table");
    const size_t bytes = (size_t)p.Nn * sizeof(long long);
    if (bytes > h->negdeg_ids.bytes && (rc = h->negdeg_ids.resize(bytes, (cudaStream_t)stream, "neg_deg_sample id list")))
      return rc;
    launch_negdeg_ids(c, p, b, b.neg_ids, h->negdeg_ids.as<long long>());
    b.neg_ids = h->negdeg_ids.as<long long>();          // from here on the step sees Cs + Ns ordinary negatives per chunk
  }
  ensure_ng_zero(h, p, w, c, false);
  // rows staged by the previous step's prefetch warps (kge_set_next_batch) are read by the fused kernels from NC / BnRaw
  const bool stageable = fused_step && p.fused && p.use_nc;
  float* const arena_nc = w.NC;
  h->pf.take_staged(*batch, stageable, p, w);
  const FusedPrefetch* pfp = nullptr;
  if ((rc = h->pf.arm_next(stageable, p, w, arena_nc, (cudaStream_t)stream, &pfp))) return rc;
  if (p.use_nc && !p.nc_staged) launch_gather_nodes(c, p, ve, b, w);      // pos_g.ndata['emb'] = entity_emb(pos_g.ndata['id'])  (general_models.py:548)
  if ((rc = (p.model == KGE_RESCAL) ? launch_rescal_prep(c, p, ve, vr, b, w) : launch_prep(c, p, ve, vr, b, w))) return rc;
  if (p.neg_deg) launch_negdeg_zero_reg(c, p, w);
  float* logdst = log4 ? log4 : h->dev_log4;
  if (p.fused) {
    launch_wbar(c, p, b.edge_weight, w);
    if ((rc = fused_launch(c, p, w, 0, b.edge_weight, fused_step ? nullptr : w.S, h->dump_v, &ve, b.neg_ids, pfp))) return rc;
    if ((rc = fused_launch(c, p, w, 1, b.edge_weight, nullptr,
                           h->dump_v ? h->dump_v + (size_t)p.B * p.Ns : nullptr, &ve, b.neg_ids, pfp))) return rc;
  } else {
    if ((rc = run_score(h, c, p, w))) return rc;
    if (p.neg_deg) launch_negdeg_mask_scores(c, p, w);
    launch_wbar(c, p, b.edge_weight, w);
    launch_loss_rows(c, p, w.pos, w.S, b.edge_weight, w);
    if (p.neg_deg) launch_negdeg_mask_coef(c, p, w);
    launch_colsum(c, p, w);
    if (use_umma(h, p)) {
      if ((rc = umma_grad(c, p, w, false))) return rc;
      if ((rc = umma_grad(c, p, w, true))) return rc;
    } else {
      launch_grad_a(c, p, w);
      launch_grad_b(c, p, w);
    }
    if (p.neg_deg) launch_negdeg_scatter(c, p, ve, b, w);
  }
  if (p.model == KGE_RESCAL) launch_rescal_chain(c, p, ve, vr, b, w);
  else launch_chain(c, p, ve, vr, b, w);
  // deferred relations into the caller's buffers: a chain that left per-edge rows (RESCAL) has them summed here, so
  // that the begin call fills the buffers for every model
  if (fused_step && p.rel_deferred && !p.rel_dense && h->ext_rg) launch_rel_grad_dense(c, p, b, w, h->ext_rg, h->ext_rgs);
  // 3-call API: the log scalars are due now; fused step: the update kernel reduces them (it also produces the unique
  // nodes' share of the regulariser when NC is skipped)
  if (!fused_step) launch_reduce_log(c, p, b.edge_weight, w, logdst, true);
  KGE_CUDA_OK(cudaGetLastError());
  h->last_p = p; h->last_w = w; h->last_b = b; h->last_ent = ve; h->last_rel = vr; h->have_last = true;
  h->ng_dirty = true;
  return KGE_OK;
}

KGE_API int kge_forward_backward(kge_handle_t h, const kge_step_cfg_t* cfg, const kge_table_t* ent, const kge_table_t* rel,
                         const kge_batch_t* batch, float* log4, void* stream) {
  return forward_backward_impl(h, cfg, ent, rel, batch, log4, stream, false);
}

static int update_impl(kge_handle_t h, const kge_step_cfg_t* cfg, const kge_table_t* ent, const kge_table_t* rel,
                       const kge_batch_t* batch, float* log4, void* stream) {
  if (!h) return fail(KGE_ERR_INVALID_ARG, "handle is null");
  if (!h->have_last) return fail(KGE_ERR_INVALID_ARG, "kge_update without a preceding kge_forward_backward");
  StepParams p;
  int rc = make_params(cfg, batch ? batch->n_nodes : 0, &p);
  if (rc) return rc;
  if ((rc = check_batch(batch, p))) return rc;
  if (p.B != h->last_p.B || p.Nn != h->last_p.Nn || p.U != h->last_p.U || p.model != h->last_p.model)
    return fail(KGE_ERR_INVALID_ARG, "kge_update cfg/batch differ from the preceding kge_forward_backward");
  TableView ve, vr;
  if ((rc = make_view(ent, &ve, "entity"))) return rc;
  if ((rc = make_view(rel, &vr, "relation"))) return rc;
  DeviceGuard g(h->device);
  StepParams q = h->last_p;       // the schedule flags (fused / use_nc / rel_dense / rel_deferred) of the forward pass
  q.lr = cfg->lr;
  BatchView b = bview(batch);
  if (q.neg_deg) b.neg_ids = h->negdeg_ids.as<long long>();     // the list the forward pass built (Cs + Ns ids per chunk)
  if ((rc = launch_update(lctx(h, stream), q, ve, vr, b, h->last_w, log4, b.edge_weight))) return rc;
  KGE_CUDA_OK(cudaGetLastError());
  h->ng_dirty = false;
  h->have_last = false;   // gradients consumed (NG re-zeroed, like `self.trace = []`, tensor_models.py:362)
  return KGE_OK;
}

KGE_API int kge_update(kge_handle_t h, const kge_step_cfg_t* cfg, const kge_table_t* ent, const kge_table_t* rel,
               const kge_batch_t* batch, void* stream) {
  return update_impl(h, cfg, ent, rel, batch, nullptr, stream);
}

// The two halves of kge_step_fused, for callers that put a collective between them (multi-GPU: all-reduce of the
// relation gradient sums while the entity update runs).
KGE_API int kge_step_fused_begin(kge_handle_t h, const kge_step_cfg_t* cfg, const kge_table_t* ent, const kge_table_t* rel,
                         const kge_batch_t* batch, void* stream) {
  if (!h) return fail(KGE_ERR_INVALID_ARG, "handle is null");
  return forward_backward_impl(h, cfg, ent, rel, batch, nullptr, stream, true);
}
KGE_API int kge_step_fused_end(kge_handle_t h, const kge_step_cfg_t* cfg, const kge_table_t* ent, const kge_table_t* rel,
                       const kge_batch_t* batch, float* log4, void* stream) {
  if (!h) return fail(KGE_ERR_INVALID_ARG, "handle is null");
  return update_impl(h, cfg, ent, rel, batch, log4 ? log4 : h->dev_log4, stream);
}

// Announce the batch of the NEXT kge_step_fused_begin: its table rows are copied by the spare warps of this step's fused
// kernels (sharded tables: the NVLink latency of step k+1 hides behind the tensor-core work of step k).
KGE_API int kge_set_next_batch(kge_handle_t h, const kge_batch_t* next, int64_t n_neg) {
  if (!h) return fail(KGE_ERR_INVALID_ARG, "handle is null");
  if (!next) { h->pf.armed = false; h->pf.ready = false; return KGE_OK; }      // also drops rows already staged
  if (!next->node_ids || !next->neg_ids || n_neg <= 0 || (next->n_nodes < 0 && !next->n_nodes_dev) || next->n_nodes == 0)
    return fail(KGE_ERR_INVALID_ARG, "kge_set_next_batch: node_ids / neg_ids / counts missing");
  h->pf.next = *next;
  h->pf.next_nneg = n_neg;
  h->pf.armed = true;
  return KGE_OK;
}

// Fused schedule (one GPU, supported shape): k_prep -> k_fused<P> -> k_fused<N> -> k_chain -> k_update = 5 launches.
KGE_API int kge_step_fused(kge_handle_t h, const kge_step_cfg_t* cfg, const kge_table_t* ent, const kge_table_t* rel,
                   const kge_batch_t* batch, float* log4, void* stream) {
  if (!h) return fail(KGE_ERR_INVALID_ARG, "handle is null");
  int rc = forward_backward_impl(h, cfg, ent, rel, batch, log4, stream, true);
  if (rc) return rc;
  return update_impl(h, cfg, ent, rel, batch, log4 ? log4 : h->dev_log4, stream);
}

KGE_API int kge_step_fused_host(kge_handle_t h, const kge_step_cfg_t* cfg, const kge_table_t* ent, const kge_table_t* rel,
                        const kge_batch_t* bh, float* log4_host, void* stream) {
  if (!h) return fail(KGE_ERR_INVALID_ARG, "handle is null");
  if (!cfg || !bh) return fail(KGE_ERR_INVALID_ARG, "cfg/batch is null");
  if (!bh->node_ids || !bh->head_local || !bh->tail_local || !bh->rel_ids || !bh->neg_ids)
    return fail(KGE_ERR_INVALID_ARG, "batch has null index arrays");
  if (cfg->batch <= 0 || cfg->chunk_size <= 0 || cfg->neg_sample_size <= 0 || cfg->batch % cfg->chunk_size)
    return fail(KGE_ERR_INVALID_ARG, "bad batch/chunk sizes");
  DeviceGuard g(h->device);
  cudaStream_t st = (cudaStream_t)stream;
  const long long B = cfg->batch, Nn = B / cfg->chunk_size * cfg->neg_sample_size, U = bh->n_nodes;
  if (U <= 0 || U > 2 * B) return fail(KGE_ERR_INVALID_ARG, "n_nodes out of range");
  // staging layout: node_ids [U] | head_local, tail_local, rel_ids [B] | neg_ids [Nn] | 256-byte aligned edge_weight [B]
  const void* src[6] = {bh->node_ids, bh->head_local, bh->tail_local, bh->rel_ids, bh->neg_ids, bh->edge_weight};
  const size_t len[6] = {(size_t)U * 8, (size_t)B * 8, (size_t)B * 8, (size_t)B * 8, (size_t)Nn * 8,
                         bh->edge_weight ? (size_t)B * 4 : 0};
  size_t off[6] = {0};
  for (int i = 1; i < 5; ++i) off[i] = off[i - 1] + len[i - 1];
  off[5] = align_up(off[4] + len[4]);
  const size_t end = len[5] ? off[5] + len[5] : off[4] + len[4];
  const size_t bytes = off[5] + align_up(len[5]) + 256;
  if (bytes > h->dev_stage.bytes) {
    int rc;
    if ((rc = h->pin.resize(bytes + bytes / 2, st, "host staging buffer")) ||
        (rc = h->dev_stage.resize(bytes + bytes / 2, st, "device staging buffer")))
      return rc;
  }
  char* const dev = h->dev_stage.as<char>();
  // Fast path: the caller's arrays are page-locked (e.g. torch pinned tensors) -> DMA straight from them.
  auto is_pinned = [](const void* p) {
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return false; }
    return a.type == cudaMemoryTypeHost;
  };
  bool direct = true;
  for (int i = 0; i < 6 && direct; ++i) direct = !len[i] || is_pinned(src[i]);
  if (direct) {
    for (int i = 0; i < 6; ++i)
      if (len[i]) cudaMemcpyAsync(dev + off[i], src[i], len[i], cudaMemcpyHostToDevice, st);
    KGE_CUDA_OK(cudaGetLastError());
  } else {
    // the previous step's H2D copy must have drained before the library's pinned buffer is overwritten
    KGE_CUDA_OK(cudaStreamSynchronize(st));
    for (int i = 0; i < 6; ++i)
      if (len[i]) memcpy(h->pin.as<char>() + off[i], src[i], len[i]);
    KGE_CUDA_OK(cudaMemcpyAsync(dev, h->pin.p, end, cudaMemcpyHostToDevice, st));
  }
  kge_batch_t bd{};
  bd.node_ids = (const int64_t*)(dev + off[0]); bd.n_nodes = U;
  bd.head_local = (const int64_t*)(dev + off[1]);
  bd.tail_local = (const int64_t*)(dev + off[2]);
  bd.rel_ids = (const int64_t*)(dev + off[3]);
  bd.neg_ids = (const int64_t*)(dev + off[4]);
  bd.edge_weight = len[5] ? (const float*)(dev + off[5]) : nullptr;
  int rc = kge_step_fused(h, cfg, ent, rel, &bd, h->dev_log4, stream);
  if (rc) return rc;
  if (log4_host) KGE_CUDA_OK(cudaMemcpyAsync(log4_host, h->dev_log4, 4 * sizeof(float), cudaMemcpyDeviceToHost, st));
  return KGE_OK;
}

KGE_API int kge_sync(kge_handle_t h, void* stream) {
  if (!h) return fail(KGE_ERR_INVALID_ARG, "handle is null");
  DeviceGuard g(h->device);
  KGE_CUDA_OK(cudaStreamSynchronize((cudaStream_t)stream));
  return KGE_OK;
}

KGE_API int kge_debug_read(kge_handle_t h, int which, float* out, int64_t n_floats, void* stream) {
  if (!h || !out) return fail(KGE_ERR_INVALID_ARG, "null argument");
  if (!h->have_last) return fail(KGE_ERR_INVALID_ARG, "no forward_backward result to read");
  const StepParams& p = h->last_p;
  const StepWs& w = h->last_w;
  DeviceGuard g(h->device);
  const float* src = nullptr;
  long long n = 0;
  switch (which) {
    case KGE_BUF_POS_SCORE: src = w.pos; n = p.B; break;
    case KGE_BUF_NEG_SCORE: src = w.S; n = p.B * p.Ns; break;
    case KGE_BUF_NEG_GRAD: src = w.Bn; n = p.Nn * p.D; break;
    case KGE_BUF_REL_GRAD: src = w.GR; n = p.B * (long long)p.Dr; break;
    case KGE_BUF_NODE_GRAD:
      n = p.U * p.D;
      if (n_floats != n) return fail(KGE_ERR_INVALID_ARG, "expected %lld floats, got %lld", n, (long long)n_floats);
      launch_node_grad_with_reg(lctx(h, stream), p, h->last_ent, h->last_b, w, out);
      KGE_CUDA_OK(cudaGetLastError());
      return KGE_OK;
    default: return fail(KGE_ERR_INVALID_ARG, "unknown buffer %d", which);
  }
  if (n_floats != n) return fail(KGE_ERR_INVALID_ARG, "expected %lld floats, got %lld", n, (long long)n_floats);
  KGE_CUDA_OK(cudaMemcpyAsync(out, src, (size_t)n * sizeof(float), cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  return KGE_OK;
}

// ---- device-side sampler ----------------------------------------------------------------------
struct kge_sampler {
  kge_context* h = nullptr;
  kge::SamplerParams base{};
  char* mem = nullptr;           // [2 buffers of index arrays | hash table]
  size_t buf_stride = 0;         // bytes between the two index buffers
  int32_t neg_sample_size = 0;
};

KGE_API int kge_sampler_create(kge_handle_t h, const int64_t* heads, const int64_t* rels, const int64_t* tails, int64_t n_edges,
                       int64_t n_entities, int64_t batch, int32_t neg_sample_size, uint64_t seed, kge_sampler_t* out) {
  if (!h || !out) return fail(KGE_ERR_INVALID_ARG, "null argument");
  *out = nullptr;
  if (!heads || !rels || !tails) return fail(KGE_ERR_INVALID_ARG, "edge arrays are null");
  if (batch <= 0 || neg_sample_size <= 0 || n_entities <= 0) return fail(KGE_ERR_INVALID_ARG, "batch / neg_sample_size / n_entities must be positive");
  if (batch % neg_sample_size != 0 && batch >= neg_sample_size)
    return fail(KGE_ERR_INVALID_ARG, "batch %lld is not a multiple of neg_sample_size %d (utils.get_compatible_batch_size)", (long long)batch, neg_sample_size);
  if (n_edges < batch) return fail(KGE_ERR_INVALID_ARG, "fewer edges (%lld) than batch (%lld)", (long long)n_edges, (long long)batch);
  if (2 * batch >= (1ll << 30)) return fail(KGE_ERR_UNSUPPORTED, "batch too large for the sampler's hash table");
  DeviceGuard g(h->device);
  kge_sampler* s = new (std::nothrow) kge_sampler();
  if (!s) return fail(KGE_ERR_NOMEM, "out of host memory");
  s->h = h;
  s->neg_sample_size = neg_sample_size;
  const long long B = batch, C = batch >= neg_sample_size ? batch / neg_sample_size : 1, Nn = C * neg_sample_size;
  int hb = 1;
  while ((1ull << (2 * hb)) < (unsigned long long)n_edges) ++hb;
  long long H = 1;
  while (H < 4 * B) H <<= 1;
  // per buffer: head, rel, tail [B] | neg [Nn] | nodes [2B] | hl, tl [B] | n_nodes [1 (+pad)]
  const size_t per_buf = align_up((size_t)(7 * B + Nn + 2) * 8);
  const size_t table = align_up((size_t)H * 8) + 2 * align_up((size_t)H * 4) + align_up((size_t)2 * B * 4);
  if (cudaMalloc(&s->mem, 2 * per_buf + table) != cudaSuccess) { cudaGetLastError(); delete s; return fail(KGE_ERR_NOMEM, "cudaMalloc for the sampler failed"); }
  s->buf_stride = per_buf;
  kge::SamplerParams& p = s->base;
  p.heads = (const long long*)heads; p.rels = (const long long*)rels; p.tails = (const long long*)tails;
  p.n_edges = n_edges; p.n_entities = n_entities; p.B = B; p.Nn = Nn; p.seed = seed; p.half_bits = hb;
  char* t = s->mem + 2 * per_buf;
  p.tkey = (unsigned long long*)t; t += align_up((size_t)H * 8);
  p.tpos = (int*)t; t += align_up((size_t)H * 4);
  p.tloc = (int*)t; t += align_up((size_t)H * 4);
  p.flags = (int*)t;
  p.hmask = (int)(H - 1);
  // empty table: keys ~0, positions INT_MAX (k_sample_reset restores this after every step)
  if (cudaMemset(p.tkey, 0xff, (size_t)H * 8) != cudaSuccess || cudaMemset(p.tpos, 0x7f, (size_t)H * 4) != cudaSuccess) {
    cudaGetLastError(); cudaFree(s->mem); delete s; return fail(KGE_ERR_CUDA, "cudaMemset failed");
  }
  // 0x7f7f7f7f is what the memset leaves in tpos: larger than any position (< 2^30), like the INT_MAX the reset writes
  *out = s;
  return KGE_OK;
}

KGE_API int kge_sampler_destroy(kge_sampler_t s) {
  if (!s) return KGE_OK;
  DeviceGuard g(s->h->device);
  cudaDeviceSynchronize();
  if (s->mem) cudaFree(s->mem);
  delete s;
  return KGE_OK;
}

KGE_API int kge_sampler_sample(kge_sampler_t s, int64_t step, kge_batch_t* out, int32_t* neg_head_out, void* stream) {
  if (!s || !out) return fail(KGE_ERR_INVALID_ARG, "null argument");
  if (step < 0) return fail(KGE_ERR_INVALID_ARG, "step < 0");
  DeviceGuard g(s->h->device);
  kge::SamplerParams p = s->base;
  long long* b = (long long*)(s->mem + (size_t)(step & 1) * s->buf_stride);
  p.o_head = b; p.o_rel = b + p.B; p.o_tail = b + 2 * p.B; p.o_neg = b + 3 * p.B;
  p.o_nodes = b + 3 * p.B + p.Nn; p.o_hl = p.o_nodes + 2 * p.B; p.o_tl = p.o_hl + p.B; p.o_n_nodes = p.o_tl + p.B;
  launch_sampler(lctx(s->h, stream), p, (long long)step);
  KGE_CUDA_OK(cudaGetLastError());
  memset(out, 0, sizeof(*out));
  out->node_ids = (const int64_t*)p.o_nodes; out->n_nodes = -1; out->n_nodes_dev = (const int64_t*)p.o_n_nodes;
  out->head_local = (const int64_t*)p.o_hl; out->tail_local = (const int64_t*)p.o_tl;
  out->rel_ids = (const int64_t*)p.o_rel; out->neg_ids = (const int64_t*)p.o_neg; out->edge_weight = nullptr;
  out->head_ids = (const int64_t*)p.o_head; out->tail_ids = (const int64_t*)p.o_tail;
  if (neg_head_out) *neg_head_out = (int32_t)(step & 1);
  return KGE_OK;
}

// ---- multi-GPU support ------------------------------------------------------------------------
KGE_API int kge_set_relation_mode(kge_handle_t h, int deferred) {
  if (!h) return fail(KGE_ERR_INVALID_ARG, "handle is null");
  h->rel_deferred = deferred ? 1 : 0;
  return KGE_OK;
}

KGE_API int kge_set_relation_buffers(kge_handle_t h, float* rg, float* rgs) {
  if (!h) return fail(KGE_ERR_INVALID_ARG, "handle is null");
  if ((rg == nullptr) != (rgs == nullptr)) return fail(KGE_ERR_INVALID_ARG, "rg and rgs must both be given or both be null");
  h->ext_rg = rg;
  h->ext_rgs = rgs;
  return KGE_OK;
}

KGE_API int kge_rel_grad_dense(kge_handle_t h, float* rg, float* rgs, void* stream) {
  if (!h || !rg || !rgs) return fail(KGE_ERR_INVALID_ARG, "null argument");
  if (!h->have_last || !h->last_p.rel_deferred)
    return fail(KGE_ERR_INVALID_ARG, "kge_rel_grad_dense needs a preceding kge_forward_backward in deferred relation mode");
  DeviceGuard g(h->device);
  launch_rel_grad_dense(lctx(h, stream), h->last_p, h->last_b, h->last_w, rg, rgs);
  KGE_CUDA_OK(cudaGetLastError());
  return KGE_OK;
}

KGE_API int kge_rel_apply_dense(kge_handle_t h, const kge_table_t* rel, float* rg, float* rgs, float lr, void* stream) {
  if (!h || !rg || !rgs) return fail(KGE_ERR_INVALID_ARG, "null argument");
  TableView vr;
  int rc = make_view(rel, &vr, "relation");
  if (rc) return rc;
  DeviceGuard g(h->device);
  launch_rel_apply_dense(lctx(h, stream), vr, rg, rgs, lr);
  KGE_CUDA_OK(cudaGetLastError());
  return KGE_OK;
}

KGE_API int kge_device_alloc(kge_handle_t h, int64_t bytes, void** out) {
  if (!h || !out || bytes <= 0) return fail(KGE_ERR_INVALID_ARG, "bad argument");
  DeviceGuard g(h->device);
  cudaError_t e = cudaMalloc(out, (size_t)bytes);
  if (e != cudaSuccess) { cudaGetLastError(); return fail(KGE_ERR_NOMEM, "cudaMalloc(%lld) failed: %s", (long long)bytes, cudaGetErrorString(e)); }
  return KGE_OK;
}

KGE_API int kge_device_free(kge_handle_t h, void* p) {
  if (!h) return fail(KGE_ERR_INVALID_ARG, "handle is null");
  DeviceGuard g(h->device);
  KGE_CUDA_OK(cudaFree(p));
  return KGE_OK;
}

KGE_API int kge_ipc_export(kge_handle_t h, const void* dev_ptr, uint8_t handle_out[64], int64_t* offset_out) {
  if (!h || !dev_ptr || !handle_out || !offset_out) return fail(KGE_ERR_INVALID_ARG, "null argument");
  DeviceGuard g(h->device);
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
  CUdeviceptr base = 0;
  size_t size = 0;
  // resolved through the runtime so that the library does not link libcuda (it must load on CPU-only hosts)
  typedef CUresult (*get_range_fn)(CUdeviceptr*, size_t*, CUdeviceptr);
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult qres;
  KGE_CUDA_OK(cudaGetDriverEntryPoint("cuMemGetAddressRange", &fn, cudaEnableDefault, &qres));
  if (!fn || qres != cudaDriverEntryPointSuccess) return fail(KGE_ERR_CUDA, "cuMemGetAddressRange not available");
  CUresult r = ((get_range_fn)fn)(&base, &size, (CUdeviceptr)dev_ptr);
  if (r != CUDA_SUCCESS) return fail(KGE_ERR_CUDA, "cuMemGetAddressRange failed (%d)", (int)r);
  cudaIpcMemHandle_t hd;
  KGE_CUDA_OK(cudaIpcGetMemHandle(&hd, (void*)base));
  memcpy(handle_out, &hd, 64);
  *offset_out = (int64_t)((CUdeviceptr)dev_ptr - base);
  return KGE_OK;
}

KGE_API int kge_ipc_open(kge_handle_t h, const uint8_t handle[64], int64_t offset, void** out) {
  if (!h || !handle || !out) return fail(KGE_ERR_INVALID_ARG, "null argument");
  DeviceGuard g(h->device);
  cudaIpcMemHandle_t hd;
  memcpy(&hd, handle, 64);
  void* base = nullptr;
  KGE_CUDA_OK(cudaIpcOpenMemHandle(&base, hd, cudaIpcMemLazyEnablePeerAccess));
  *out = (char*)base + offset;
  return KGE_OK;
}

// ---- peer-shareable shard memory (CUDA virtual memory management) --------------------------------------------------
// A cudaMalloc range opened in another process through cudaIpcOpenMemHandle is mapped there with small pages: random
// row reads over a large peer shard then miss the reader's TLB on every row.  cuMemCreate allocations exported as POSIX file
// descriptors map with 2 MiB pages on both sides.
namespace {
struct Vmm {
  CUresult (*create)(CUmemGenericAllocationHandle*, size_t, const CUmemAllocationProp*, unsigned long long) = nullptr;
  CUresult (*release)(CUmemGenericAllocationHandle) = nullptr;
  CUresult (*exporth)(void*, CUmemGenericAllocationHandle, CUmemAllocationHandleType, unsigned long long) = nullptr;
  CUresult (*importh)(CUmemGenericAllocationHandle*, void*, CUmemAllocationHandleType) = nullptr;
  CUresult (*reserve)(CUdeviceptr*, size_t, size_t, CUdeviceptr, unsigned long long) = nullptr;
  CUresult (*addrfree)(CUdeviceptr, size_t) = nullptr;
  CUresult (*map)(CUdeviceptr, size_t, size_t, CUmemGenericAllocationHandle, unsigned long long) = nullptr;
  CUresult (*unmap)(CUdeviceptr, size_t) = nullptr;
  CUresult (*setaccess)(CUdeviceptr, size_t, const CUmemAccessDesc*, size_t) = nullptr;
  CUresult (*gran)(size_t*, const CUmemAllocationProp*, CUmemAllocationGranularity_flags) = nullptr;
  bool ok = false;
};
const Vmm& vmm() {
  static Vmm v = [] {
    Vmm t;
    cudaDriverEntryPointQueryResult q;
    auto get = [&](const char* name, void** fn) {
      return cudaGetDriverEntryPoint(name, fn, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess && *fn;
    };
    t.ok = get("cuMemCreate", (void**)&t.create) && get("cuMemRelease", (void**)&t.release) &&
           get("cuMemExportToShareableHandle", (void**)&t.exporth) && get("cuMemImportFromShareableHandle", (void**)&t.importh) &&
           get("cuMemAddressReserve", (void**)&t.reserve) && get("cuMemAddressFree", (void**)&t.addrfree) &&
           get("cuMemMap", (void**)&t.map) && get("cuMemUnmap", (void**)&t.unmap) && get("cuMemSetAccess", (void**)&t.setaccess) &&
           get("cuMemGetAllocationGranularity", (void**)&t.gran);
    return t;
  }();
  return v;
}
CUmemAllocationProp shard_prop(int device) {
  CUmemAllocationProp prop;
  memset(&prop, 0, sizeof(prop));
  prop.type = CU_MEM_ALLOCATION_TYPE_PINNED;
  prop.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
  prop.location.id = device;
  prop.requestedHandleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
  return prop;
}
int shard_map(kge_handle_t h, CUmemGenericAllocationHandle mh, size_t size, size_t gran, void** out) {
  const Vmm& v = vmm();
  CUdeviceptr va = 0;
  CUresult r = v.reserve(&va, size, gran, 0, 0);
  if (r != CUDA_SUCCESS) return fail(KGE_ERR_NOMEM, "cuMemAddressReserve(%zu) failed (%d)", size, (int)r);
  r = v.map(va, size, 0, mh, 0);
  if (r != CUDA_SUCCESS) { v.addrfree(va, size); return fail(KGE_ERR_CUDA, "cuMemMap failed (%d)", (int)r); }
  CUmemAccessDesc acc;
  memset(&acc, 0, sizeof(acc));
  acc.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
  acc.location.id = h->device;
  acc.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
  r = v.setaccess(va, size, &acc, 1);
  if (r != CUDA_SUCCESS) { v.unmap(va, size); v.addrfree(va, size); return fail(KGE_ERR_CUDA, "cuMemSetAccess failed (%d): no peer path between the GPUs?", (int)r); }
  *out = (void*)va;
  return KGE_OK;
}
size_t shard_round(int device, int64_t bytes, size_t* gran_out) {
  CUmemAllocationProp prop = shard_prop(device);
  size_t gran = 2u << 20;
  vmm().gran(&gran, &prop, CU_MEM_ALLOC_GRANULARITY_RECOMMENDED);
  if (gran < (2u << 20)) gran = 2u << 20;
  *gran_out = gran;
  return ((size_t)bytes + gran - 1) / gran * gran;
}
}  // namespace

KGE_API int kge_shard_alloc(kge_handle_t h, int64_t bytes, void** out, int* fd_out) {
  if (!h || !out || !fd_out || bytes <= 0) return fail(KGE_ERR_INVALID_ARG, "bad argument");
  DeviceGuard g(h->device);
  KGE_CUDA_OK(cudaFree(0));
  if (!vmm().ok) return fail(KGE_ERR_CUDA, "CUDA virtual memory management entry points not available");
  const Vmm& v = vmm();
  size_t gran = 0;
  const size_t size = shard_round(h->device, bytes, &gran);
  CUmemAllocationProp prop = shard_prop(h->device);
  CUmemGenericAllocationHandle mh;
  CUresult r = v.create(&mh, size, &prop, 0);
  if (r != CUDA_SUCCESS) return fail(KGE_ERR_NOMEM, "cuMemCreate(%zu) failed (%d)", size, (int)r);
  int fd = -1;
  r = v.exporth(&fd, mh, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR, 0);
  if (r != CUDA_SUCCESS) { v.release(mh); return fail(KGE_ERR_CUDA, "cuMemExportToShareableHandle failed (%d)", (int)r); }
  int rc = shard_map(h, mh, size, gran, out);
  v.release(mh);                 // the mapping (and the fd, until closed) keep the allocation alive
  if (rc) { close(fd); return rc; }
  *fd_out = fd;
  return KGE_OK;
}

KGE_API int kge_shard_import(kge_handle_t h, int fd, int64_t bytes, void** out) {
  if (!h || !out || fd < 0 || bytes <= 0) return fail(KGE_ERR_INVALID_ARG, "bad argument");
  DeviceGuard g(h->device);
  KGE_CUDA_OK(cudaFree(0));
  if (!vmm().ok) return fail(KGE_ERR_CUDA, "CUDA virtual memory management entry points not available");
  const Vmm& v = vmm();
  size_t gran = 0;
  const size_t size = shard_round(h->device, bytes, &gran);
  CUmemGenericAllocationHandle mh;
  CUresult r = v.importh(&mh, (void*)(uintptr_t)fd, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR);
  if (r != CUDA_SUCCESS) return fail(KGE_ERR_CUDA, "cuMemImportFromShareableHandle failed (%d)", (int)r);
  int rc = shard_map(h, mh, size, gran, out);
  v.release(mh);
  return rc;
}

KGE_API int kge_shard_free(kge_handle_t h, void* ptr, int64_t bytes) {
  if (!h || !ptr || bytes <= 0) return fail(KGE_ERR_INVALID_ARG, "bad argument");
  DeviceGuard g(h->device);
  if (!vmm().ok) return fail(KGE_ERR_CUDA, "CUDA virtual memory management entry points not available");
  size_t gran = 0;
  const size_t size = shard_round(h->device, bytes, &gran);
  KGE_CUDA_OK(cudaDeviceSynchronize());
  CUresult r = vmm().unmap((CUdeviceptr)ptr, size);
  if (r != CUDA_SUCCESS) return fail(KGE_ERR_CUDA, "cuMemUnmap failed (%d)", (int)r);
  vmm().addrfree((CUdeviceptr)ptr, size);
  return KGE_OK;
}

}  // extern "C"
