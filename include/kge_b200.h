/*
 * kge_b200.h -- C ABI of libkge_b200.so: the H100-native (sm_90a) replacement for the
 * per-step hot path of awslabs/dgl-ke's `dglke_train`:
 *
 *   ExternalEmbedding gather  ->  score_func over 1 positive + chunk-shared negatives
 *   ->  logsigmoid (+ self-adversarial) loss gradient  ->  row-sparse Adagrad scatter update
 *
 * The reference has no native layer (it is pure Python on top of PyTorch ATen); each entry
 * point below therefore cites the *Python* function it replaces, with file:line relative to
 * python/dglke of awslabs/dgl-ke.  The host side (dgl-ke_b200/dglke_b200) binds this header with
 * ctypes and mirrors the reference's KEModel / score_func / ExternalEmbedding surface.
 *
 * Conventions
 *   - every data pointer is a CUDA device pointer unless the name ends in `_host`
 *   - tables are fp32 row-major [num_rows, dim]; all indices are int64
 *   - calls enqueue work on `stream` (a cudaStream_t passed as void*) and return immediately;
 *     the *_host variants copy through pinned staging buffers owned by the handle
 *   - return value: 0 = KGE_OK, negative = kge_status; nothing throws across the ABI;
 *     kge_last_error() returns a thread-local description of the last failure
 *   - a handle is bound to one device and is not thread-safe; use one handle per GPU/process
 *   - chunk layout: chunk c owns positives [c*chunk_size, (c+1)*chunk_size) and negative ids
 *     [c*neg_sample_size, (c+1)*neg_sample_size); only same-chunk pairs are scored
 *     (dataloader/sampler.py:459-512)
 */
#ifndef KGE_B200_H_
#define KGE_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define KGE_API __attribute__((visibility("default")))
#else
#define KGE_API
#endif

#define KGE_ABI_VERSION 4
#define KGE_MAX_SHARDS 8

typedef enum {
  KGE_OK = 0,
  KGE_ERR_INVALID_ARG = -1,   /* null pointer, negative size, batch not a multiple of chunk_size ... */
  KGE_ERR_UNSUPPORTED = -2,   /* model/dim combination this build does not implement              */
  KGE_ERR_CUDA = -3,          /* a CUDA runtime call failed; see kge_last_error()                  */
  KGE_ERR_NOMEM = -4,         /* workspace allocation failed                                       */
  KGE_ERR_NO_DEVICE = -5      /* no usable sm_90 device                                            */
} kge_status;

/* models/general_models.py:238-258 (model_name -> score_func) */
typedef enum {
  KGE_TRANSE_L1 = 0,
  KGE_TRANSE_L2 = 1,
  KGE_DISTMULT = 2,
  KGE_COMPLEX = 3,
  KGE_RESCAL = 4,
  KGE_ROTATE = 5
} kge_model_t;

/* One row-range shard of an embedding table.  `emb`/`state_sum` may be peer-mapped pointers to
 * another GPU's HBM (NVLink): kernels then load / red.add over the fabric.
 * Replaces ExternalEmbedding.emb / .state_sum (models/pytorch/tensor_models.py:210-238). */
typedef struct {
  float* emb;          /* [row_end-row_begin, dim] */
  float* state_sum;    /* [row_end-row_begin]      */
  int64_t row_begin, row_end;
  int32_t dim;
  int32_t device;
} kge_shard_t;

/* A table = n_shards contiguous row ranges of equal size ceil(num_rows / n_shards). */
typedef struct {
  const kge_shard_t* shards;   /* host array */
  int32_t n_shards;
  int64_t num_rows;
  int32_t dim;
} kge_table_t;

/* Per-step configuration.  Mirrors the fields KEModel/LossGenerator/ExternalEmbedding read from
 * `args` (models/general_models.py:208-236,572-576; models/pytorch/loss.py:41-62;
 * models/pytorch/tensor_models.py:320). */
typedef struct {
  int32_t model;            /* kge_model_t */
  int32_t entity_dim;       /* D_e: fp32 per entity row                                   */
  int32_t relation_dim;     /* D_r: fp32 per relation row (RESCAL: rel_dim * entity_dim)  */
  float gamma;              /* TransE / RotatE margin                                     */
  float emb_init;           /* (gamma + 2) / hidden_dim; RotatE phase scale               */
  float lr;                 /* Adagrad learning rate                                      */
  float reg_coef;           /* regularization_coef (0 disables)                           */
  int32_t reg_norm;         /* regularization_norm p (0 disables)                         */
  int32_t adversarial;      /* -adv: self-adversarial negative weighting                  */
  float adv_temperature;
  int32_t neg_head;         /* 1: this step corrupts heads, 0: tails (sampler.py:853-859) */
  int64_t batch;            /* B positives; must equal num_chunks * chunk_size            */
  int32_t chunk_size;       /* positives per chunk                                        */
  int32_t neg_sample_size;  /* negatives per chunk                                        */
  /* ABI 3: the loss criterion (models/pytorch/loss.py:10-62).  Logistic and BCE are the Logsigmoid criterion written
   * differently (softplus(-l*s) == -logsigmoid(l*s); BCE with labels 1 / 0 likewise) and share its kernels; the
   * reference's BCE evaluates log(sigmoid(s)) and overflows to inf beyond |s| ~ 88 where this library stays finite. */
  int32_t loss_genre;       /* kge_loss_t                                                 */
  float margin;             /* Hinge: max(0, margin - label * score)                      */
  int32_t pairwise;         /* -pw: criterion(pos_i - neg_ij, 1), mean over all pairs (Hinge / Logistic only; the
                             * self-adversarial weighting does not apply, loss.py:76-80)   */
  /* ABI 4: --neg_deg_sample (models/general_models.py:396-403,417-424,429-432): the chunk's own corrupted-side rows are
   * scored as chunk_size extra negatives in front of the sampled ones (score of a positive against its own row forced
   * to 0, gradients of the extra columns go to the positive nodes).  neg_sample_size stays the SAMPLED count and
   * batch.neg_ids holds num_chunks * neg_sample_size ids; the negative-score matrix (kge_debug_read) is
   * [batch, chunk_size + neg_sample_size].  Training entry points only, single-shard tables. */
  int32_t neg_deg_sample;
} kge_step_cfg_t;
typedef enum { KGE_LOSS_LOGSIGMOID = 0, KGE_LOSS_HINGE = 1, KGE_LOSS_LOGISTIC = 2, KGE_LOSS_BCE = 3 } kge_loss_t;

/* The sampled batch, exactly the tensors KEModel.forward pulls out of (pos_g, neg_g).  The kernels index the tables
 * with these ids as given: an id outside [0, num_rows) is undefined behaviour (the reference's tensor indexing raises
 * IndexError); the Python layer validates them when KGE_B200_CHECK_IDS=1.
 * (models/general_models.py:376-427,548-549):
 *   node_ids   = pos_g.ndata['id']              int64[n_nodes]  unique entity ids of the batch
 *   head_local,
 *   tail_local = pos_g.all_edges(order='eid')   int64[batch]    indices into node_ids
 *   rel_ids    = pos_g.edata['id']              int64[batch]
 *   neg_ids    = neg_g.ndata['id'][neg_g.head_nid | tail_nid]   int64[num_chunks*neg_sample_size]
 *   edge_weight= pos_g.edata['impts']           float[batch] or NULL */
typedef struct {
  const int64_t* node_ids;
  int64_t n_nodes;
  const int64_t* head_local;
  const int64_t* tail_local;
  const int64_t* rel_ids;
  const int64_t* neg_ids;
  const float* edge_weight;
  const int64_t* n_nodes_dev;  /* device-side node count (kge_sampler_sample): used when n_nodes < 0; node_ids then
                                  has room for 2*batch entries */
  const int64_t* head_ids;     /* optional: global entity ids of the edges' endpoints (= node_ids[head_local],   */
  const int64_t* tail_ids;     /*   node_ids[tail_local]); saves the kernels one dependent index load per row     */
} kge_batch_t;

typedef struct kge_context* kge_handle_t;

KGE_API int kge_abi_version(void);
KGE_API const char* kge_last_error(void);

/* Creates the per-device context (workspace, pinned staging, SM count).  `device` is a CUDA
 * ordinal.  Fails with KGE_ERR_NO_DEVICE when no sm_90 GPU is present -- there is no CPU path. */
KGE_API int kge_create(int device, kge_handle_t* out);
KGE_API int kge_destroy(kge_handle_t h);

/* --- unfused pieces: one per reference function, used by the plugin classes and parity tests --- */

/* ExternalEmbedding.__call__  (tensor_models.py:270-302): out[i,:] = table[idx[i],:]  (bit exact) */
KGE_API int kge_gather(kge_handle_t h, const kge_table_t* table, const int64_t* idx, int64_t n,
               float* out, void* stream);

/* score_func.edge_func (score_fun.py:54-59,229-235,297-307,387-394,460-472) on gathered rows
 * head/tail [n, D_e], rel [n, D_r] -> out[n] */
KGE_API int kge_score_pos(kge_handle_t h, const kge_step_cfg_t* cfg, const float* head, const float* rel,
                  const float* tail, int64_t n, float* out, void* stream);

/* score_func.create_neg(neg_head)(heads, relations, tails, C, Cs, Ns)
 * (score_fun.py:91-108,268-286,345-376,427-449,512-554).
 *   cfg->neg_head == 0: heads/rel are the positives' rows [batch,.], tails = negative rows [C*Ns, D_e]
 *   cfg->neg_head == 1: heads = negative rows [C*Ns, D_e], tails/rel the positives' rows
 * out: [C, chunk_size, neg_sample_size] */
KGE_API int kge_score_neg(kge_handle_t h, const kge_step_cfg_t* cfg, const float* heads, const float* rel,
                  const float* tails, float* out, void* stream);

/* LossGenerator.get_total_loss, Logsigmoid criterion, + d loss / d score (loss.py:69-98).
 * pos [batch], neg [batch, Ns], w [batch] or NULL.  dpos [batch], dneg [batch, Ns],
 * log4 = {pos_loss, neg_loss, loss, 0} (device) */
KGE_API int kge_loss_grad(kge_handle_t h, const kge_step_cfg_t* cfg, const float* pos, const float* neg,
                  const float* w, float* dpos, float* dneg, float* log4, void* stream);

/* One trace entry of ExternalEmbedding.update (tensor_models.py:316-361; identical math in
 * async_update :154-175 and kvserver.py:41-50): state_sum[idx] += mean(g^2) for every row
 * (duplicates accumulate), THEN emb[idx] += -lr * g / (sqrt(state_sum[idx]) + 1e-10). */
KGE_API int kge_adagrad(kge_handle_t h, const kge_table_t* table, const int64_t* idx, const float* grad,
                int64_t n, float lr, void* stream);

/* --- the step -------------------------------------------------------------------------------- */

/* KEModel.forward + loss.backward() (general_models.py:529-578, train_pytorch.py:141-145):
 * gathers, scores, loss, and all gradients; leaves the gradients in the handle's workspace and
 * writes log4 = {pos_loss, neg_loss, loss (without reg), regularization} to device memory. */
KGE_API int kge_forward_backward(kge_handle_t h, const kge_step_cfg_t* cfg, const kge_table_t* ent,
                         const kge_table_t* rel, const kge_batch_t* batch, float* log4, void* stream);

/* KEModel.update (general_models.py:580-588): applies the gradients of the last
 * kge_forward_backward: entity entries [unique positive nodes, negatives], then relations. */
KGE_API int kge_update(kge_handle_t h, const kge_step_cfg_t* cfg, const kge_table_t* ent,
               const kge_table_t* rel, const kge_batch_t* batch, void* stream);

/* forward + backward + update in one call (train_pytorch.py:141-152). */
KGE_API int kge_step_fused(kge_handle_t h, const kge_step_cfg_t* cfg, const kge_table_t* ent,
                   const kge_table_t* rel, const kge_batch_t* batch, float* log4, void* stream);

/* kge_step_fused in two halves, for callers that put a collective between them (multi-GPU: the relation all-reduce
 * overlaps the entity update): begin = gather .. k_chain, end = k_update (+ log scalars into log4). */
KGE_API int kge_step_fused_begin(kge_handle_t h, const kge_step_cfg_t* cfg, const kge_table_t* ent,
                         const kge_table_t* rel, const kge_batch_t* batch, void* stream);
KGE_API int kge_step_fused_end(kge_handle_t h, const kge_step_cfg_t* cfg, const kge_table_t* ent,
                       const kge_table_t* rel, const kge_batch_t* batch, float* log4, void* stream);

/* Software pipelining for sharded tables (the reference's --async_update staleness, tensor_models.py:136-175: the rows a
 * step reads may lag the updates of the step before it).  kge_set_next_batch announces the batch of the NEXT
 * kge_step_fused_begin; the spare warps of this step's fused kernels then copy that batch's unique-node rows and negative
 * rows (peer loads over NVLink) into staging buffers while the tensor cores work, and the next begin -- called with
 * exactly that batch: same device arrays, contents unchanged -- skips its own gathers.  One announcement serves one step;
 * a begin with any other batch simply ignores the staged rows.  Only node_ids / n_nodes(_dev) / neg_ids of `next` are
 * read; n_neg = num_chunks * neg_sample_size of the next step.  next = NULL cancels the announcement and drops
 * rows already staged.  The staging buffers are allocated
 * on first use (not during stream capture). */
KGE_API int kge_set_next_batch(kge_handle_t h, const kge_batch_t* next, int64_t n_neg);

/* Same as kge_step_fused but the batch index arrays (and edge weights) are HOST memory, as they
 * come out of the sampler.  Pageable arrays are staged through the handle's pinned buffer (they may be
 * reused as soon as the call returns); page-locked arrays (cudaHostAlloc / torch pin_memory) are DMA'd
 * directly and must stay unchanged until kge_sync.  The four log scalars are copied back to log4_host
 * (D2H) on `stream` -- call kge_sync before reading them. */
KGE_API int kge_step_fused_host(kge_handle_t h, const kge_step_cfg_t* cfg, const kge_table_t* ent,
                        const kge_table_t* rel, const kge_batch_t* batch_host, float* log4_host,
                        void* stream);
KGE_API int kge_sync(kge_handle_t h, void* stream);

/* --- device-side sampler (replaces DGL's EdgeSampler on the training path: dataloader/sampler.py:376-419 create_sampler,
 *     :459-512 chunk layout, :823-876 tail/head alternation) -------------------------------------------------------------
 * heads/rels/tails: the (partition's) edge list in device memory, owned by the caller.  Step k takes the k-th batch of
 * the current epoch's random permutation (a fresh one per epoch, ragged tail dropped), draws num_chunks * neg_sample_size
 * corrupting entities uniformly with replacement, and builds the positive graph's node list (distinct endpoints in order of
 * first appearance) + local endpoints -- all in device memory, counter based (seed, step): dglke_b200/sampler.py holds
 * the same integer arithmetic in numpy and produces bit-identical arrays.  Even steps corrupt tails, odd steps heads. */
typedef struct kge_sampler* kge_sampler_t;
KGE_API int kge_sampler_create(kge_handle_t h, const int64_t* heads, const int64_t* rels, const int64_t* tails,
                       int64_t n_edges, int64_t n_entities, int64_t batch, int32_t neg_sample_size, uint64_t seed,
                       kge_sampler_t* out);
KGE_API int kge_sampler_destroy(kge_sampler_t s);
/* Fills *batch_out with device pointers into the sampler's storage (two buffers, alternating with `step`; valid until the
 * next-but-one call), n_nodes = -1 and n_nodes_dev set; *neg_head_out = step & 1. */
KGE_API int kge_sampler_sample(kge_sampler_t s, int64_t step, kge_batch_t* batch_out, int32_t* neg_head_out, void* stream);

/* --- filtered ranking of evaluation queries (KEModel.forward_test's rank, general_models.py:462-485) -----------------
 *   rank_q = 1 + #{ j : S[q, j] >= pos[q] (IEEE: a NaN never counts) and candidate j is not a known triple of q }
 * over the score tiles of kge_score_neg, tile by tile, without a [queries, candidates] mask.
 *
 * The known triples of one corruption side: keys[i] = kept_entity * n_rel + rel, sorted; vals[i] = the corrupted-side
 * entity, sorted and distinct within each key (device arrays).  Corrupting heads, the kept side is the tail. */
typedef struct {
  const int64_t* keys;
  const int32_t* vals;
  int64_t n_keys;
  int64_t n_rel;
} kge_filter_t;

/* Adds one score tile's hits to cnt[Q] (int64, zeroed by the caller once per batch of queries).
 *   S [Q, ld]: N columns used;  pos [Q]: the positives' scores
 *   kept [Q], rel [Q]: each query's kept-side entity and relation (read only with a filter)
 *   cand == NULL: column j is entity base + j (a block of rows of one shard);
 *   cand != NULL: cand [Q / chunk, N] int64 ids, query q ranks against row q / chunk (chunked sampled candidates)
 *   filter == NULL or filter->n_keys == 0: raw ranks */
KGE_API int kge_rank_count(kge_handle_t h, const float* S, int64_t ld, int64_t Q, int64_t N, const float* pos,
                           int64_t base, const int64_t* cand, int64_t chunk, const int64_t* kept, const int64_t* rel,
                           const kge_filter_t* filter, int64_t* cnt, void* stream);
/* rank = cnt + 1: written to rank_out [Q] (int64) unless NULL, and {sum 1/r, sum r, #(r<=1), #(r<=3), #(r<=10), Q}
 * added to acc [6] (device doubles, caller-owned; reduced in a fixed order, so the sums do not depend on timing). */
KGE_API int kge_rank_finish(kge_handle_t h, const int64_t* cnt, int64_t Q, int64_t* rank_out, double* acc,
                            void* stream);

/* --- running top-K lists over score tiles (link prediction, ScoreInfer.topK of models/infer.py) ----------------------
 * Merges score tile S [Q, ld] (N columns used) into G running lists of K entries:
 *   row q feeds list g = qgroup[q] (0 <= g < G); the rows of one list are consecutive within a call
 *   element (q, j) has key = qoff[q] + (cbase + j) * cstride (qoff >= 0, cbase >= 0, cstride >= 1); keys are distinct
 *   top_score [G, K], top_key [G, K]: caller-owned device arrays, initialised once to -inf / -1 (empty slots)
 * After the call every list holds the K best of (itself U the tile's elements of its rows) in the strict order
 * score descending, then key ascending; fewer than K elements seen leaves trailing -inf / -1 slots.  A NaN score never
 * enters, a -inf one does.  The result is the host sort of the same fp32 scores, bit for bit, whatever the launch
 * geometry or timing.  1 <= K <= KGE_TOPK_MAX, else KGE_ERR_UNSUPPORTED (K > max) / KGE_ERR_INVALID_ARG (K < 1).
 * Workspace: about Q * ceil(N / 4096) * (12 K + 4) + 4 G bytes, kept on the handle (it grows, synchronising the stream
 * once, when a call needs more). */
#define KGE_TOPK_MAX 1024
KGE_API int kge_topk(kge_handle_t h, const float* S, int64_t ld, int64_t Q, int64_t N, const int64_t* qgroup,
                     const int64_t* qoff, int64_t cbase, int64_t cstride, int32_t K, int64_t G, float* top_score,
                     int64_t* top_key, void* stream);

/* --- embedding similarity (dglke_emb_sim: EmbSimInfer of models/infer.py:216-343, the *_dist functions of
 *     models/pytorch/tensor_models.py:59-100), fp32 rows x, y of `dim` floats ------------------------------------------
 *   COSINE       x.y / (|x| |y|)                      (a zero row gives NaN, as in the reference)
 *   L2           -|x - y|_2                           (difference form: x = y gives exactly -0.0)
 *   L1           -|x - y|_1                           (likewise)
 *   DOT          x.y
 *   EXT_JACCARD  x.y / (|x|^2 + |y|^2 - x.y)          (|x|^2 is the square of the fp32 norm) */
typedef enum { KGE_SIM_COSINE = 0, KGE_SIM_L2 = 1, KGE_SIM_L1 = 2, KGE_SIM_DOT = 3, KGE_SIM_EXT_JACCARD = 4 } kge_sim_t;
/* out [nL, nR] (contiguous) = sim(left[i], right[j]); left [nL, dim], right [nR, dim] row-major (any alignment).
 * DOT / COSINE / EXT_JACCARD: 3xTF32 tensor-core GEMM with the function applied to the accumulator; L1 / L2: fp32
 * CUDA-core tiles.  1 <= dim <= 160000 (a RESCAL relation row at hidden 400).  The GEMM functions keep TF32 copies of
 * both blocks on the handle: about 8 (nL + nR) ceil(dim / 32) * 32 bytes (it grows, synchronising the stream once, when
 * a call needs more). */
KGE_API int kge_sim_tile(kge_handle_t h, int32_t sim, const float* left, int64_t nL, const float* right, int64_t nR,
                         int32_t dim, float* out, void* stream);
/* out [n] = sim(left[i], right[i]) (the reference's pw=True) */
KGE_API int kge_sim_pairs(kge_handle_t h, int32_t sim, const float* left, const float* right, int64_t n, int32_t dim,
                          float* out, void* stream);

/* --- introspection (parity tests read the traced gradients the way the reference exposes
 *     `data.grad` of each trace entry, tensor_models.py:318) ---------------------------------- */
typedef enum {
  KGE_BUF_POS_SCORE = 0,   /* [batch]                                     */
  KGE_BUF_NEG_SCORE = 1,   /* [batch, Ns]  (overwritten by backward coefficients after the loss) */
  KGE_BUF_NODE_GRAD = 2,   /* [n_nodes, D_e]  d loss / d unique positive node rows (incl. reg)   */
  KGE_BUF_NEG_GRAD = 3,    /* [C*Ns, D_e]                                                        */
  KGE_BUF_REL_GRAD = 4     /* [batch, D_r]                                                       */
} kge_buffer_t;
/* Copies a workspace buffer of the last kge_forward_backward to `out` (device). For
 * KGE_BUF_NEG_SCORE call with cfg of that step *before* kge_update. */
KGE_API int kge_debug_read(kge_handle_t h, int which, float* out, int64_t n_floats, void* stream);

/* Number of kernels the library has launched on this handle since creation. */
KGE_API int64_t kge_launch_count(kge_handle_t h);
/* Per-launch device timing: when enabled, every kernel the library launches on this handle is
 * bracketed by CUDA events on the launching stream (<= 64 records; enable resets the record set).
 * kge_profile_read synchronises the device, writes the kernel names ('|' separated) and their
 * durations in milliseconds, returns the record count and starts a new record set. */
KGE_API int kge_profile_enable(kge_handle_t h, int on);
KGE_API int kge_profile_read(kge_handle_t h, char* names, int names_len, float* ms, int max_records);
/* Selects the contraction engine: 0 = fp32 CUDA-core tiles, 1 = wgmma 3xTF32 tensor-core tiles
 * (bilinear models), -1 = library default. */
KGE_API int kge_set_engine(kge_handle_t h, int engine);

/* Selects the contraction schedule of the bilinear / L2 models: -1 (default) or 1 = the fused wgmma kernel
 * (score -> loss -> coefficients in registers -> gradient GEMM, kge_fused.cu) whenever the chunk shape fits its register budget
 * (chunk_size, neg_sample_size <= 240), 0 = separate GEMM / loss kernels. */
KGE_API int kge_set_fused(kge_handle_t h, int mode);
/* Test hook: when non-null, the fused kernel also writes its backward coefficients dL/dneg_ij (/ dist_ij for
 * TransE_l2) to coef_dump: [batch, Ns] as seen by the positive-side pass, then [C*Ns, chunk_size] as recomputed by the
 * negative-side pass (device memory, 2 * batch * Ns floats). */
KGE_API int kge_debug_set_dump(kge_handle_t h, float* coef_dump);

/* --- multi-GPU: row-range sharded entity table over peer-mapped HBM, replicated relation table ---
 * Replaces --mix_cpu_gpu's host-pinned shared table (general_models.py:230-231, train.py:92-95):
 * each rank allocates its shard, exports it with kge_ipc_export, opens every peer's shard with
 * kge_ipc_open and passes all shards in kge_table_t; kernels then gather with peer loads and
 * scatter with system-scope red.add over NVLink.
 * Relation rows are replicated; in deferred mode the step leaves per-edge relation gradients in the
 * workspace, kge_rel_grad_dense sums them per relation into rg [num_rel, D_r] / rgs [num_rel]
 * (sum of mean(g^2)), the host all-reduces both with NCCL, and kge_rel_apply_dense applies the same
 * Adagrad update on every replica and zeroes the buffers. */
KGE_API int kge_set_relation_mode(kge_handle_t h, int deferred);
/* Deferred mode, fused step: caller-owned dense buffers rg [num_rel, D_r] and rgs [num_rel] (zero between steps) that
 * kge_step_fused_begin sums the per-relation gradients / mean squares into (no kge_rel_grad_dense; RESCAL, whose
 * chain kernel writes per-edge rows, gets one extra summing launch); the caller all-reduces them and calls
 * kge_rel_apply_dense.  NULL, NULL = off. */
KGE_API int kge_set_relation_buffers(kge_handle_t h, float* rg, float* rgs);
KGE_API int kge_rel_grad_dense(kge_handle_t h, float* rg, float* rgs, void* stream);
KGE_API int kge_rel_apply_dense(kge_handle_t h, const kge_table_t* rel, float* rg, float* rgs, float lr, void* stream);
KGE_API int kge_device_alloc(kge_handle_t h, int64_t bytes, void** out);
KGE_API int kge_device_free(kge_handle_t h, void* p);
KGE_API int kge_ipc_export(kge_handle_t h, const void* dev_ptr, uint8_t handle_out[64], int64_t* offset_out);
KGE_API int kge_ipc_open(kge_handle_t h, const uint8_t handle[64], int64_t offset, void** out);
/* Shard memory for LARGE tables (what dglke_b200.dist uses): CUDA virtual-memory-management allocations, shared between
 * the ranks as POSIX file descriptors (pass them over a Unix socket, SCM_RIGHTS) and mapped with 2 MiB pages on the owner
 * and on every peer.  kge_ipc_open maps a peer's cudaMalloc range with small pages, and random row reads over a shard of
 * tens of GB then miss the reader's TLB on every row.
 *   kge_shard_alloc   allocate `bytes` (rounded up to the mapping granularity) on the handle's device, map it read/write,
 *                     return the pointer and a file descriptor the caller passes to peers and then close()s
 *   kge_shard_import  map the allocation behind a received descriptor read/write on the handle's device (same `bytes`)
 *   kge_shard_free    unmap (owner or importer side); the memory is released when the last mapping and descriptor go */
KGE_API int kge_shard_alloc(kge_handle_t h, int64_t bytes, void** out, int* fd_out);
KGE_API int kge_shard_import(kge_handle_t h, int fd, int64_t bytes, void** out);
KGE_API int kge_shard_free(kge_handle_t h, void* ptr, int64_t bytes);

#ifdef __cplusplus
}
#endif
#endif /* KGE_B200_H_ */
