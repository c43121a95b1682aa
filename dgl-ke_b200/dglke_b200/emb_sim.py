"""Embedding similarity on the GPU: `python -m dglke_b200.emb_sim` (the reference's dglke_emb_sim, infer_emb_sim.py and
EmbSimInfer.topK of models/infer.py), with the same flags and the same output file.

The reference builds the whole |L| x |R| score matrix on the host and argsorts it.  Here kge_sim_tile computes one tile
of similarities at a time and kge_topk merges it into running top-K lists on the GPU, so nothing larger than a tile
exists.  Similarity functions (models/pytorch/tensor_models.py:59-100), in fp32:
  cosine        x.y / (|x| |y|)            dot           x.y
  l2            -|x - y|_2                 ext_jaccard   x.y / (|x|^2 + |y|^2 - x.y)
  l1            -|x - y|_1
dot, cosine and ext_jaccard run as a 3xTF32 tensor-core GEMM with the function applied to the accumulator; l1 and l2 run
on fp32 CUDA-core tiles in difference form, so a row against itself scores exactly -0.0, as in the reference.

Exec modes as tiles (Plan below; it runs without a GPU).  The left rows are always the queries (tile rows):
  pairwise     kge_sim_pairs over batches of (l_i, r_i): one [1, n] tile per batch, key i, one list
  all          every (l_i, r_j): key i |R| + j (the reference's flat index), one list
  batch_left   one list per left row, key i |R| + j; a left batch's lists live on the GPU only while that batch runs
A side that is every row ('*' in --format) is read from the table in place, in blocks of rows; a given list is gathered
block by block (it may repeat ids: each position is an element of its own).  Query batches and right blocks are sized by
evaluate.EVAL_BUDGET_BYTES, on a library handle of this module's own.  Lists are ordered by score descending, then key
ascending; this is the reference's argsort wherever scores do not tie (its argsort is not stable, so ties have no
reference order).

Deliberate differences from the reference:
  - pairwise with lists of unequal length is refused (the reference slices the right list by the left list's length);
  - when a list has fewer than K pairs, only those are returned and written: every column of a list has one length (the
    reference's batch_left returns a length-K np.full column beside shorter ones);
  - reading a list strips only the line ending (the reference's id[:-1] cuts the last character of a final line that
    has no newline);
  - a NaN score (cosine of a zero row; ext_jaccard of two zero rows) never enters a list (the reference's descending
    argsort ranks NaN first);
  - a table that is not float32 is converted to float32 (training writes float32);
  - bad input is refused up front: an unknown format, function or mode, a 1-D --emb_file, ids out of range, --topK
    outside [1, KGE_TOPK_MAX], and --gpu -1 (there is no CPU path)."""
import argparse
import ctypes as C
import sys

import numpy as np
import torch

from . import _lib
from .engine import DeviceTable
from .evaluate import EVAL_BUDGET_BYTES
from .predict import NO_GPU, read_id_list, read_mapping, read_name_list

FORMATS = ("l_r", "l_*", "*_r", "*")
EXEC_MODES = ("pairwise", "all", "batch_left")
SIM_FUNCS = tuple(_lib.SIM_IDS)
QUERY_BATCH = 2048              # left rows per similarity tile
MAX_DIM = 160000                # kge_sim_tile's limit: a RESCAL relation row at hidden 400


class ArgParser(argparse.ArgumentParser):
    """The reference's infer_emb_sim.ArgParser: the same flags, types and defaults."""

    def __init__(self):
        super(ArgParser, self).__init__()
        A = self.add_argument
        A("--mfile", type=str, default=None, help="id<TAB>name mapping file (with --raw_data)")
        A("--emb_file", type=str, default=None, help="numpy file of the embeddings, [rows, dim]")
        A("--format", type=str, help="which lists are given: l_r (left and right), l_* (left; every row is a right "
          "object), *_r (right; every row is a left object), * (every row on both sides)")
        A("--data_files", type=str, default=None, nargs="+", help="the given lists, left first")
        A("--raw_data", default=False, action="store_true",
          help="the lists hold names, mapped through --mfile (and back in the output)")
        A("--exec_mode", type=str, default="all", help="pairwise | all | batch_left")
        A("--topK", type=int, default=10, help="how many results are returned (per left object in batch_left)")
        A("--sim_func", type=str, default="cosine", help="cosine | l2 | l1 | dot | ext_jaccard")
        A("--output", type=str, default="result.tsv", help="the result file")
        A("--gpu", type=int, default=-1, help="the GPU to use; -1 (CPU) is refused")


# ------------------------------------------------------------------------------------------------------------- inputs
def read_lists(fmt, data_files, raw_data=False, mfile=None):
    """(left, right) id arrays, None where the format has '*', and the id -> name map (None without --raw_data)."""
    if fmt not in FORMATS:
        raise SystemExit("Unsupported format {}".format(fmt))
    given = [fmt[0] != "*", fmt[-1] != "*"]
    data_files = data_files or []
    if len(data_files) != sum(given):
        raise SystemExit("format %s needs %d data files, got %d" % (fmt, sum(given), len(data_files)))
    i2e = None
    if raw_data:
        if mfile is None:
            raise SystemExit("When using RAW ID through --raw_data, mfile should be provided.")
        e2i, i2e = read_mapping(mfile)
    files = iter(data_files)
    out = [None if not g else (read_name_list(next(files), e2i) if raw_data else read_id_list(next(files)))
           for g in given]
    return out[0], out[1], i2e


def check_ids(left, right, n):
    """Refuses a list id outside [0, n) (the reference's tensor indexing raises IndexError, or wraps a negative id)."""
    for lst, what in ((left, "left"), (right, "right")):
        if lst is not None and len(lst) and (np.min(lst) < 0 or np.max(lst) >= n):
            raise SystemExit("a %s id is outside [0, %d)" % (what, n))


def load_table(path):
    """The --emb_file table as a float32 [rows, dim] array."""
    emb = np.load(path)
    if emb.ndim != 2:
        raise SystemExit("--emb_file %s holds a %d-D array: a table of [rows, dim] embeddings is needed" % (path, emb.ndim))
    return emb.astype(np.float32, copy=False)


# ------------------------------------------------------------------------------------------------------------ planning
class Plan:
    """How one exec mode maps onto similarity tiles, for nL left and nR right objects.
      n_lists           G, the number of result lists
      cstride           key step from one right object to the next (1)
      queries(b, e)     the left rows [b, e) in tile order as (positions, list, qoff); a list's rows are consecutive
    Key of (left row i, right position j) = qoff_i + j = i nR + j (pairwise: one [1, n] row, key i)."""

    def __init__(self, exec_mode, nL, nR):
        if exec_mode not in EXEC_MODES:
            raise SystemExit("unknow execution mode type {}".format(exec_mode))
        if exec_mode == "pairwise" and nL != nR:
            raise SystemExit("For pairwise execution mode, left and right lists should have same length (%d vs %d)"
                             % (nL, nR))
        self.mode, self.nL, self.nR, self.cstride = exec_mode, nL, nR, 1
        self.n_lists = nL if exec_mode == "batch_left" else 1

    def queries(self, b, e):
        i = np.arange(b, e, dtype=np.int64)
        g = i if self.mode == "batch_left" else np.zeros_like(i)
        return i, g, i * self.nR

    def decode(self, keys):
        """Positions (i, j) in the left and right lists of keys."""
        keys = np.asarray(keys, dtype=np.int64)
        if self.mode == "pairwise":
            return keys, keys
        return keys // self.nR, keys % self.nR


# ----------------------------------------------------------------------------------------------------------- execution
class EmbSim:
    """Top-K embedding similarity over one table (numpy or torch, converted to float32) on one GPU.  Runs on a library
    handle of its own, on the current stream of `device`."""

    def __init__(self, emb, device=0, budget=EVAL_BUDGET_BYTES, query_batch=QUERY_BATCH):
        emb = torch.as_tensor(emb)
        if emb.dim() != 2:
            raise SystemExit("the embedding table must be 2-D [rows, dim], got shape %s" % (tuple(emb.shape),))
        if not 1 <= emb.shape[1] <= MAX_DIM:
            raise SystemExit("embedding width %d is outside [1, %d]" % (emb.shape[1], MAX_DIM))
        self.budget, self.query_batch = budget, query_batch
        self.h = _lib.Handle(device)
        self.device, self.lib = self.h.device, self.h.lib
        self.n, self.dim = emb.shape
        # rows are stored zero-padded to whole 16-byte vectors (kge_gather copies float4s); zero columns change none of
        # the five functions
        self.ld = -(-self.dim // 4) * 4
        free, total = torch.cuda.mem_get_info(self.device)
        need = self.n * self.ld * 4
        if need + 2 * budget > free:
            raise SystemExit("the table needs %.2f GB on cuda:%d, which has %.2f GB free of %.2f GB: similarity needs the "
                             "table on one GPU" % (need / 1e9, self.device.index, free / 1e9, total / 1e9))
        self.emb = torch.zeros((self.n, self.ld), dtype=torch.float32, device=self.device)
        self.emb[:, :self.dim] = emb.to(self.device, torch.float32)
        self._t = DeviceTable.from_tensors(self.emb, torch.zeros(self.n, device=self.device))

    def close(self):
        self.h.close()

    def _rows(self, ids, b, e):
        """Rows [b, e) of a side: the table's own rows in place (ids None), else the gathered rows of ids[b:e]."""
        if ids is None:
            return C.c_void_p(self.emb.data_ptr() + b * self.ld * 4), None
        out = torch.empty((e - b, self.ld), dtype=torch.float32, device=self.device)
        _lib.check(self.lib.kge_gather(self.h.raw, self._t.ref(), ids[b:e].data_ptr(), e - b, out.data_ptr(),
                                       self.h.stream()))
        return C.c_void_p(out.data_ptr()), out

    def block_rows(self, Q, K):
        """Right rows per tile: the tile's column, a gathered row, its TF32 copies and norm, and kge_topk's survivors."""
        per_row = 4 * Q + 4 * self.ld + 8 * 32 * (-(-self.ld // 32)) + 4 + (Q * (12 * K + 4)) // 4096 + 1
        return max(1, self.budget // per_row)

    def tiles(self, plan, sim, L, R, K):
        """Yields (S [Q, n] device tile, left rows [b, e), qgroup, qoff, cbase) of every tile, in order; S is reused.
        L, R: device id tensors (or None: every row of the table, in id order)."""
        sid, stream = _lib.SIM_IDS[sim], self.h.stream()
        if plan.mode == "pairwise":
            nb = max(1, min(plan.nL, self.budget // (8 * self.ld + 4)))
            S = torch.empty(nb, dtype=torch.float32, device=self.device)
            zero = torch.zeros(1, dtype=torch.int64, device=self.device)
            for b in range(0, plan.nL, nb):
                e = min(plan.nL, b + nb)
                (lp, lk), (rp, rk) = self._rows(L, b, e), self._rows(R, b, e)
                _lib.check(self.lib.kge_sim_pairs(self.h.raw, sid, lp, rp, e - b, self.ld, S.data_ptr(), stream))
                yield S[:e - b].view(1, e - b), (0, 1), zero, zero, b
            return
        Qb = min(plan.nL, self.query_batch)
        nb = min(plan.nR, self.block_rows(Qb, K))
        S = torch.empty(Qb * nb, dtype=torch.float32, device=self.device)
        for qb in range(0, plan.nL, Qb):
            qe = min(plan.nL, qb + Qb)
            Q = qe - qb
            _, g, off = plan.queries(qb, qe)
            qgroup, qoff = torch.from_numpy(g).to(self.device), torch.from_numpy(off).to(self.device)
            lp, lk = self._rows(L, qb, qe)
            for c0 in range(0, plan.nR, nb):
                n = min(nb, plan.nR - c0)
                rp, rk = self._rows(R, c0, c0 + n)
                _lib.check(self.lib.kge_sim_tile(self.h.raw, sid, lp, Q, rp, n, self.ld, S.data_ptr(), stream))
                yield S[:Q * n].view(Q, n), (qb, qe), qgroup, qoff, c0

    def topk_keys(self, plan, sim, L, R, k):
        """The raw lists, moved to the host list batch by list batch: (scores [G, K], keys [G, K]) numpy arrays, empty
        slots -inf / -1.  batch_left keeps only the current left batch's lists on the GPU."""
        K = int(k)
        if not 1 <= K <= _lib.KGE_TOPK_MAX:
            raise SystemExit("--topK %d is outside [1, %d] (KGE_TOPK_MAX)" % (K, _lib.KGE_TOPK_MAX))
        G = plan.n_lists
        out_s = np.full((G, K), -np.inf, dtype=np.float32)
        out_k = np.full((G, K), -1, dtype=np.int64)
        if plan.nL == 0 or plan.nR == 0:
            return out_s, out_k
        per_batch = plan.mode == "batch_left"
        stream = self.h.stream()
        top_s = top_k = None
        cur = None
        for S, (b, e), qgroup, qoff, cbase in self.tiles(plan, sim, L, R, K):
            if top_s is None or (per_batch and (b, e) != cur):
                if per_batch and top_s is not None:
                    out_s[cur[0]:cur[1]], out_k[cur[0]:cur[1]] = top_s.cpu().numpy(), top_k.cpu().numpy()
                n_lists = e - b if per_batch else 1
                top_s = torch.full((n_lists, K), float("-inf"), dtype=torch.float32, device=self.device)
                top_k = torch.full((n_lists, K), -1, dtype=torch.int64, device=self.device)
                cur = (b, e)
            Q, N = S.shape
            qg = qgroup - b if per_batch else qgroup
            _lib.check(self.lib.kge_topk(self.h.raw, S.data_ptr(), N, Q, N, qg.data_ptr(), qoff.data_ptr(), cbase,
                                         plan.cstride, K, top_s.shape[0], top_s.data_ptr(), top_k.data_ptr(), stream))
        if per_batch:
            out_s[cur[0]:cur[1]], out_k[cur[0]:cur[1]] = top_s.cpu().numpy(), top_k.cpu().numpy()
        else:
            out_s[:], out_k[:] = top_s.cpu().numpy(), top_k.cpu().numpy()
        return out_s, out_k

    def topk(self, left=None, right=None, exec_mode="all", k=10, sim_func="cosine"):
        """EmbSimInfer.topK: [(left ids, right ids, scores)] per list, numpy, best first (only the pairs that exist)."""
        if sim_func not in SIM_FUNCS:
            raise SystemExit("unknown similarity function %s (one of %s)" % (sim_func, ", ".join(SIM_FUNCS)))
        nL = self.n if left is None else len(left)
        nR = self.n if right is None else len(right)
        plan = Plan(exec_mode, nL, nR)
        check_ids(left, right, self.n)
        ids = [None if x is None else torch.as_tensor(np.asarray(x, dtype=np.int64)).to(self.device)
               for x in (left, right)]
        top_s, top_k = self.topk_keys(plan, sim_func, *ids, k)
        full = lambda x, n: np.arange(n, dtype=np.int64) if x is None else np.asarray(x, dtype=np.int64)
        Ln, Rn = full(left, nL), full(right, nR)
        out = []
        for g in range(plan.n_lists):
            m = top_k[g] >= 0
            i, j = plan.decode(top_k[g][m])
            out.append((Ln[i], Rn[j], top_s[g][m]))
        return out


def write_result(path, result, id2e=None):
    """infer_emb_sim.py's file: a header, then one line per pair, lists in order, each best first."""
    with open(path, "w+") as f:
        f.write("left\tright\tscore\n")
        for ll, rl, sl in result:
            for a, b, s in zip(ll.tolist(), rl.tolist(), sl.tolist()):
                if id2e is not None:
                    a, b = id2e[a], id2e[b]
                f.write("{}\t{}\t{}\n".format(a, b, s))


def main(argv=None):
    args = ArgParser().parse_args(argv)
    if args.gpu < 0:
        raise SystemExit(NO_GPU)
    if args.emb_file is None:
        raise SystemExit("emb_file should be provided for entity embeddings")
    if args.sim_func not in SIM_FUNCS:
        raise SystemExit("unknown similarity function %s (one of %s)" % (args.sim_func, ", ".join(SIM_FUNCS)))
    if args.exec_mode not in EXEC_MODES:
        raise SystemExit("unknow execution mode type {}".format(args.exec_mode))
    if not 1 <= args.topK <= _lib.KGE_TOPK_MAX:
        raise SystemExit("--topK %d is outside [1, %d] (KGE_TOPK_MAX)" % (args.topK, _lib.KGE_TOPK_MAX))
    left, right, id2e = read_lists(args.format, args.data_files, args.raw_data, args.mfile)
    emb = load_table(args.emb_file)
    check_ids(left, right, emb.shape[0])
    Plan(args.exec_mode, emb.shape[0] if left is None else len(left), emb.shape[0] if right is None else len(right))
    torch.cuda.set_device(args.gpu)
    s = EmbSim(emb, args.gpu)
    try:
        result = s.topk(left, right, args.exec_mode, args.topK, args.sim_func)
    finally:
        s.close()
    write_result(args.output, result, id2e if args.raw_data else None)
    print("Inference Done")
    print("The result is saved in {}".format(args.output))


if __name__ == "__main__":
    sys.exit(main())
