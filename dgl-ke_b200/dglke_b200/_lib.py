"""ctypes binding of libkge_b200.so (include/kge_b200.h).

There is NO fallback: if the shared library is missing, cannot be loaded, or no sm_90 GPU is
visible, every entry point raises.  The structures below mirror the C header field by field.
"""
import ctypes as C
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("KGE_B200_LIB", os.path.join(os.path.dirname(_HERE), "lib", "libkge_b200.so"))

KGE_MAX_SHARDS = 8
KGE_TOPK_MAX = 1024
SIM_IDS = {"cosine": 0, "l2": 1, "l1": 2, "dot": 3, "ext_jaccard": 4}       # kge_sim_t
MODEL_IDS = {"TransE_l1": 0, "TransE": 1, "TransE_l2": 1, "DistMult": 2, "ComplEx": 3, "RESCAL": 4, "RotatE": 5}
BUF_POS_SCORE, BUF_NEG_SCORE, BUF_NODE_GRAD, BUF_NEG_GRAD, BUF_REL_GRAD = range(5)

EXPORTS = ["kge_abi_version", "kge_last_error", "kge_create", "kge_destroy", "kge_gather", "kge_score_pos",
           "kge_score_neg", "kge_loss_grad", "kge_adagrad", "kge_forward_backward", "kge_update",
           "kge_step_fused", "kge_step_fused_begin", "kge_step_fused_end", "kge_step_fused_host", "kge_sync", "kge_debug_read", "kge_launch_count",
           "kge_set_engine", "kge_set_fused", "kge_debug_set_dump", "kge_profile_enable", "kge_profile_read", "kge_set_relation_mode", "kge_set_relation_buffers",
           "kge_rel_grad_dense", "kge_rel_apply_dense", "kge_device_alloc", "kge_device_free", "kge_ipc_export",
           "kge_ipc_open", "kge_shard_alloc", "kge_shard_import", "kge_shard_free",
           "kge_set_next_batch", "kge_sampler_create", "kge_sampler_destroy", "kge_sampler_sample",
           "kge_rank_count", "kge_rank_finish", "kge_topk", "kge_sim_tile", "kge_sim_pairs"]


class KgeError(RuntimeError):
    pass


class Shard(C.Structure):
    _fields_ = [("emb", C.c_void_p), ("state_sum", C.c_void_p), ("row_begin", C.c_int64),
                ("row_end", C.c_int64), ("dim", C.c_int32), ("device", C.c_int32)]


class Table(C.Structure):
    _fields_ = [("shards", C.POINTER(Shard)), ("n_shards", C.c_int32), ("num_rows", C.c_int64),
                ("dim", C.c_int32)]


class StepCfg(C.Structure):
    _fields_ = [("model", C.c_int32), ("entity_dim", C.c_int32), ("relation_dim", C.c_int32),
                ("gamma", C.c_float), ("emb_init", C.c_float), ("lr", C.c_float), ("reg_coef", C.c_float),
                ("reg_norm", C.c_int32), ("adversarial", C.c_int32), ("adv_temperature", C.c_float),
                ("neg_head", C.c_int32), ("batch", C.c_int64), ("chunk_size", C.c_int32),
                ("neg_sample_size", C.c_int32), ("loss_genre", C.c_int32), ("margin", C.c_float),
                ("pairwise", C.c_int32), ("neg_deg_sample", C.c_int32)]


LOSS_IDS = {"Logsigmoid": 0, "Hinge": 1, "Logistic": 2, "BCE": 3}       # kge_loss_t


class Batch(C.Structure):
    _fields_ = [("node_ids", C.c_void_p), ("n_nodes", C.c_int64), ("head_local", C.c_void_p),
                ("tail_local", C.c_void_p), ("rel_ids", C.c_void_p), ("neg_ids", C.c_void_p),
                ("edge_weight", C.c_void_p), ("n_nodes_dev", C.c_void_p), ("head_ids", C.c_void_p),
                ("tail_ids", C.c_void_p)]


class Filter(C.Structure):
    _fields_ = [("keys", C.c_void_p), ("vals", C.c_void_p), ("n_keys", C.c_int64), ("n_rel", C.c_int64)]


_lib = None


def load_library():
    """dlopen the library and declare the prototypes.  Does not touch the GPU."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise KgeError("libkge_b200.so not found at %s -- build it with `python -c 'import __graft_entry__ as g; "
                       "g.build()'` (there is no CPU/PyTorch fallback)" % LIB_PATH)
    lib = C.CDLL(LIB_PATH)
    vp, i32, i64, f32 = C.c_void_p, C.c_int32, C.c_int64, C.c_float
    P = C.POINTER
    lib.kge_abi_version.restype = C.c_int
    lib.kge_last_error.restype = C.c_char_p
    lib.kge_create.argtypes = [C.c_int, P(vp)]
    lib.kge_destroy.argtypes = [vp]
    lib.kge_gather.argtypes = [vp, P(Table), vp, i64, vp, vp]
    lib.kge_score_pos.argtypes = [vp, P(StepCfg), vp, vp, vp, i64, vp, vp]
    lib.kge_score_neg.argtypes = [vp, P(StepCfg), vp, vp, vp, vp, vp]
    lib.kge_loss_grad.argtypes = [vp, P(StepCfg), vp, vp, vp, vp, vp, vp, vp]
    lib.kge_adagrad.argtypes = [vp, P(Table), vp, vp, i64, f32, vp]
    lib.kge_forward_backward.argtypes = [vp, P(StepCfg), P(Table), P(Table), P(Batch), vp, vp]
    lib.kge_update.argtypes = [vp, P(StepCfg), P(Table), P(Table), P(Batch), vp]
    lib.kge_step_fused.argtypes = [vp, P(StepCfg), P(Table), P(Table), P(Batch), vp, vp]
    lib.kge_step_fused_begin.argtypes = [vp, P(StepCfg), P(Table), P(Table), P(Batch), vp]
    lib.kge_step_fused_end.argtypes = [vp, P(StepCfg), P(Table), P(Table), P(Batch), vp, vp]
    lib.kge_step_fused_host.argtypes = [vp, P(StepCfg), P(Table), P(Table), P(Batch), vp, vp]
    lib.kge_sync.argtypes = [vp, vp]
    lib.kge_debug_read.argtypes = [vp, C.c_int, vp, i64, vp]
    lib.kge_launch_count.argtypes = [vp]
    lib.kge_launch_count.restype = i64
    lib.kge_set_engine.argtypes = [vp, C.c_int]
    lib.kge_set_fused.argtypes = [vp, C.c_int]
    lib.kge_debug_set_dump.argtypes = [vp, vp]
    lib.kge_profile_enable.argtypes = [vp, C.c_int]
    lib.kge_profile_read.argtypes = [vp, C.c_char_p, C.c_int, P(f32), C.c_int]
    lib.kge_set_relation_mode.argtypes = [vp, C.c_int]
    lib.kge_set_relation_buffers.argtypes = [vp, vp, vp]
    lib.kge_rel_grad_dense.argtypes = [vp, vp, vp, vp]
    lib.kge_rel_apply_dense.argtypes = [vp, P(Table), vp, vp, f32, vp]
    lib.kge_device_alloc.argtypes = [vp, i64, P(vp)]
    lib.kge_device_free.argtypes = [vp, vp]
    lib.kge_ipc_export.argtypes = [vp, vp, C.c_char_p, P(i64)]
    lib.kge_ipc_open.argtypes = [vp, C.c_char_p, i64, P(vp)]
    lib.kge_shard_alloc.argtypes = [vp, i64, P(vp), P(C.c_int)]
    lib.kge_shard_import.argtypes = [vp, C.c_int, i64, P(vp)]
    lib.kge_shard_free.argtypes = [vp, vp, i64]
    lib.kge_set_next_batch.argtypes = [vp, P(Batch), i64]
    lib.kge_sampler_create.argtypes = [vp, vp, vp, vp, i64, i64, i64, i32, C.c_uint64, P(vp)]
    lib.kge_sampler_destroy.argtypes = [vp]
    lib.kge_sampler_sample.argtypes = [vp, i64, P(Batch), P(i32), vp]
    lib.kge_rank_count.argtypes = [vp, vp, i64, i64, i64, vp, i64, vp, i64, vp, vp, P(Filter), vp, vp]
    lib.kge_rank_finish.argtypes = [vp, vp, i64, vp, vp, vp]
    lib.kge_topk.argtypes = [vp, vp, i64, i64, i64, vp, vp, i64, i64, i32, i64, vp, vp, vp]
    lib.kge_sim_tile.argtypes = [vp, i32, vp, i64, vp, i64, i32, vp, vp]
    lib.kge_sim_pairs.argtypes = [vp, i32, vp, vp, i64, i32, vp, vp]
    missing = [name for name in EXPORTS if not hasattr(lib, name)]
    if missing:
        raise KgeError("libkge_b200.so at %s lacks symbols %s (stale build?)" % (LIB_PATH, missing))
    _lib = lib
    return lib


def check(rc):
    if rc != 0:
        raise KgeError("libkge_b200 error %d: %s" % (rc, load_library().kge_last_error().decode()))


def current_stream(device):
    return C.c_void_p(torch.cuda.current_stream(device).cuda_stream)


class Handle:
    """One kge_handle_t bound to one CUDA device."""

    def __init__(self, device=0):
        lib = load_library()
        if not torch.cuda.is_available():
            raise KgeError("no CUDA device: libkge_b200 is an H100 (sm_90a) library and has no CPU path")
        self.device = torch.device("cuda", device if isinstance(device, int) else device.index)
        self._h = C.c_void_p()
        check(lib.kge_create(self.device.index, C.byref(self._h)))
        self.lib = lib

    def close(self):
        if getattr(self, "_h", None) is not None and self._h:
            self.lib.kge_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def raw(self):
        return self._h

    def stream(self):
        return current_stream(self.device)

    def launch_count(self):
        return int(self.lib.kge_launch_count(self._h))

    def set_engine(self, engine):
        check(self.lib.kge_set_engine(self._h, int(engine)))

    def set_fused(self, mode):
        """-1 / 1: fused wgmma contraction kernel when the shape allows (default); 0: separate GEMM + loss kernels."""
        check(self.lib.kge_set_fused(self._h, int(mode)))

    def set_dump(self, tensor):
        """test hook: device float tensor of 2 * batch * Ns elements receiving the fused kernel's coefficients (or None)"""
        self._dump_keep = tensor
        check(self.lib.kge_debug_set_dump(self._h, C.c_void_p(tensor.data_ptr()) if tensor is not None else None))

    def profile_enable(self, on=True):
        check(self.lib.kge_profile_enable(self._h, 1 if on else 0))

    def profile_read(self):
        """[(kernel name, milliseconds)] of every launch since the last read (syncs the device)."""
        names = C.create_string_buffer(8192)
        ms = (C.c_float * 64)()
        n = self.lib.kge_profile_read(self._h, names, 8192, ms, 64)
        if n < 0:
            check(n)
        nm = names.value.decode().split("|") if n else []
        return [(nm[i], float(ms[i])) for i in range(min(n, len(nm)))]


_handles = {}


def get_handle(device=0):
    idx = device if isinstance(device, int) else (device.index or 0)
    if idx not in _handles:
        _handles[idx] = Handle(idx)
    return _handles[idx]


def make_table(shards_emb, shards_state, num_rows, dim, devices=None):
    """Build a kge_table_t from per-shard (emb_ptr, state_ptr) pairs.  `shards_emb[i]` may be a
    torch tensor (local shard) or an int device pointer (peer-mapped shard).  Returns
    (Table, keepalive)."""
    n = len(shards_emb)
    arr = (Shard * n)()
    rows_per = (num_rows + n - 1) // n
    for s in range(n):
        e, st = shards_emb[s], shards_state[s]
        arr[s].emb = e.data_ptr() if torch.is_tensor(e) else int(e)
        arr[s].state_sum = st.data_ptr() if torch.is_tensor(st) else int(st)
        arr[s].row_begin = s * rows_per
        arr[s].row_end = min(num_rows, (s + 1) * rows_per)
        arr[s].dim = dim
        arr[s].device = devices[s] if devices else 0
    t = Table(arr, n, num_rows, dim)
    return t, (arr, shards_emb, shards_state)


def make_cfg(model, entity_dim, relation_dim, gamma, emb_init, lr, reg_coef, reg_norm, adversarial,
             adv_temperature, neg_head, batch, chunk_size, neg_sample_size, loss_genre="Logsigmoid", margin=1.0,
             pairwise=False, neg_deg_sample=False):
    if model not in MODEL_IDS:
        raise KgeError("model %r is not on the accelerated hot path (supported: %s)" % (model, sorted(MODEL_IDS)))
    if loss_genre not in LOSS_IDS:
        raise ValueError("loss genre %s is not support" % loss_genre)            # loss.py:58-59
    return StepCfg(MODEL_IDS[model], entity_dim, relation_dim, gamma, emb_init, lr, reg_coef, reg_norm,
                   1 if adversarial else 0, adv_temperature, 1 if neg_head else 0, batch, chunk_size,
                   neg_sample_size, LOSS_IDS[loss_genre], float(margin), 1 if pairwise else 0, 1 if neg_deg_sample else 0)


def make_batch(node_ids, head_local, tail_local, rel_ids, neg_ids, edge_weight=None, head_ids=None, tail_ids=None):
    """Index tensors may be CUDA tensors (device ABI) or CPU tensors (host ABI); int64, contiguous.
    head_ids / tail_ids (optional, = node_ids[head_local], node_ids[tail_local]) save the kernels an index hop."""
    for t in (node_ids, head_local, tail_local, rel_ids, neg_ids):
        assert t.dtype == torch.int64 and t.is_contiguous()
    ptr = lambda t: t.data_ptr() if t is not None else None
    b = Batch(node_ids.data_ptr(), node_ids.numel(), head_local.data_ptr(), tail_local.data_ptr(),
              rel_ids.data_ptr(), neg_ids.data_ptr(), ptr(edge_weight), None, ptr(head_ids), ptr(tail_ids))
    return b, (node_ids, head_local, tail_local, rel_ids, neg_ids, edge_weight, head_ids, tail_ids)
