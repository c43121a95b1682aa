"""Link prediction from a saved checkpoint on the GPU: `python -m dglke_b200.predict` (the reference's dglke_predict,
infer_score.py and ScoreInfer.topK of models/infer.py), with the same flags and the same output file.

The reference builds the whole H x R x T score vector, copies it to the host and argsorts it.  Here the scores come
from kge_score_neg / kge_score_pos one tile at a time, and kge_topk merges each tile into running top-K lists on the GPU,
so nothing larger than a tile exists.  Keys are the reference's flat index (i |R| + j) |T| + k, with i, j, k positions in
the H, R and T lists, so a key decodes to its output row; the lists order by raw score descending, then key ascending.

Exec modes as tiles (Plan below; it runs without a GPU):
  triplet_wise                 kge_score_pos over batches of (h_i, r_i, t_i): one [1, n] tile per batch, key i, one list
  all / batch_head / batch_rel queries (h_i, r_j), the T list as candidates (columns): list 0, i or j
  batch_tail                   queries (r_j, t_k), the H list as candidates (kge_score_neg's head mode): list k,
                               column stride |R| |T|
A candidate list that is every entity ('*' in --format) is scored in place, in blocks of table rows; a given list is
gathered block by block (it may repeat ids: each position is a candidate of its own).  Query batches and blocks are
sized by evaluate.default_block_rows's workspace budget, on a library handle of this module's own.

RESCAL: kge_score_neg's tail mode computes the reference's training score h^T M_r^T t', not the inference score
h^T M_r t'.  Tail candidates therefore run in head mode against a transposed copy of the relation matrices, built once:
(M_r^T h) . t' = h^T M_r t'.  Head candidates use head mode and M_r as they are, as RESCALScore.infer does.

Score semantics (ScoreInfer.load_model): with --score_func none the model's gamma is 0 (TransE scores -|h + r - t|,
RotatE -sum |.|); with logsigmoid it is the config's gamma and logsigmoid is applied to the K selected scores (it is
monotone, so ranking on the raw score selects the same set).  A reference quirk is kept on purpose: InferModel derives
RotatE's phase scale emb_init = (gamma + 2) / hidden_dim from that gamma, so under `none` the relation phases are
r / ((2 / hidden_dim) / pi), not the trained model's; the lists agree with the reference's, not with a training-time
score.

Two deliberate differences from the reference:
  - when a list has fewer than K triples, only those are returned and written: every column of a list has one length
    (the reference's batch modes return a length-K np.full column beside shorter ones);
  - reading a list strips only the line ending (the reference's id[:-1] cuts the last character of a final line that
    has no newline).
TransR and SimplE are refused, as in training; --gpu -1 is refused (there is no CPU path)."""
import argparse
import csv
import ctypes as C
import json
import os
import sys

import numpy as np
import torch

from . import _lib
from .engine import Hyper, DeviceTable, _cfg_for
from .evaluate import EVAL_BUDGET_BYTES, default_block_rows

FORMATS = ("h_r_t", "h_r_*", "h_*_t", "*_r_t", "h_*_*", "*_r_*", "*_*_t")
EXEC_MODES = ("triplet_wise", "all", "batch_head", "batch_rel", "batch_tail")
QUERY_BATCH = 2048              # queries per score tile
NO_GPU = "dglke_b200 needs --gpu: the hot path is an H100 CUDA library without a CPU fallback"


class ArgParser(argparse.ArgumentParser):
    """The reference's infer_score.ArgParser: the same flags, types and defaults."""

    def __init__(self):
        super(ArgParser, self).__init__()
        A = self.add_argument
        A("--model_path", type=str, default="ckpts", help="the directory of the saved model (config.json, *.npy)")
        A("--format", type=str, help="which of the head, relation and tail lists are given: " + ", ".join(FORMATS) +
          "; '*' means every entity or relation")
        A("--data_files", type=str, default=None, nargs="+", help="the given lists, in h, r, t order")
        A("--raw_data", default=False, action="store_true",
          help="the lists hold names, mapped through --entity_mfile / --rel_mfile (and back in the output)")
        A("--exec_mode", type=str, default="all", help="triplet_wise | all | batch_head | batch_rel | batch_tail")
        A("--topK", type=int, default=10, help="how many results are returned (per list in the batch modes)")
        A("--score_func", type=str, default="none", help="none: score = x; logsigmoid: score = log(sigmoid(x))")
        A("--output", type=str, default="result.tsv", help="the result file")
        A("--entity_mfile", type=str, default=None, help="entity id mapping file (with --raw_data)")
        A("--rel_mfile", type=str, default=None, help="relation id mapping file (with --raw_data)")
        A("--gpu", type=int, default=-1, help="the GPU to use; -1 (CPU) is refused")


# ------------------------------------------------------------------------------------------------------------- inputs
def _lines(path):
    """The lines of a list file with only the line ending stripped (a last line without one is kept whole)."""
    with open(path, "r") as f:
        return [ln[:-1] if ln.endswith("\n") else ln for ln in f]


def read_id_list(path):
    return np.asarray([int(x) for x in _lines(path)], dtype=np.int64)


def read_mapping(path):
    """id<TAB>name per line (entities.dict / relations.dict) -> (name -> id, id -> name)."""
    n2i, i2n = {}, {}
    with open(path, "r") as f:
        for row in csv.reader(f, delimiter="\t"):
            n2i[row[1]] = int(row[0])
            i2n[int(row[0])] = row[1]
    return n2i, i2n


def read_name_list(path, name2id):
    return np.asarray([name2id[x] for x in _lines(path)], dtype=np.int64)


def read_lists(fmt, data_files, raw_data=False, entity_mfile=None, rel_mfile=None):
    """(head, rel, tail) id arrays, None where the format has '*', and (id2e, id2r) maps (None without --raw_data)."""
    if fmt not in FORMATS:
        raise SystemExit("Unsupported format {}".format(fmt))
    given = [c != "*" for c in fmt.split("_")]
    data_files = data_files or []
    if len(data_files) != sum(given):
        raise SystemExit("format %s needs %d data files, got %d" % (fmt, sum(given), len(data_files)))
    maps = (None, None)
    if raw_data:
        if entity_mfile is None or rel_mfile is None:
            raise SystemExit("When using RAW ID through --raw_data, entity_mfile and rel_mfile should be provided.")
        (e2i, i2e), (r2i, i2r) = read_mapping(entity_mfile), read_mapping(rel_mfile)
        maps = (i2e, i2r)
    files = iter(data_files)
    out = []
    for side, g in zip("hrt", given):
        if not g:
            out.append(None)
        elif raw_data:
            out.append(read_name_list(next(files), r2i if side == "r" else e2i))
        else:
            out.append(read_id_list(next(files)))
    return out[0], out[1], out[2], maps


# --------------------------------------------------------------------------------------------------------- checkpoint
def checkpoint_files(model_path, dataset, model_name):
    """The two .npy tables of a checkpoint.  KEModel saves a `--model_name TransE` run under TransE_l2 while config.json
    says TransE (the multi-GPU path saves it under TransE): either name is found."""
    names = [model_name] + (["TransE_l2"] if model_name == "TransE" else [])
    for n in names:
        e = os.path.join(model_path, "%s_%s_entity.npy" % (dataset, n))
        r = os.path.join(model_path, "%s_%s_relation.npy" % (dataset, n))
        if os.path.exists(e) and os.path.exists(r):
            return e, r
    raise SystemExit("no %s_{%s}_{entity,relation}.npy in %s" % (dataset, ",".join(names), model_path))


def load_checkpoint(model_path):
    """(config dict, entity table, relation table) as numpy float32."""
    with open(os.path.join(model_path, "config.json"), "r") as f:
        config = json.load(f)
    if config["model_name"] in ("TransR", "SimplE"):
        raise SystemExit("model %s is not supported by dglke_b200 (TransR and SimplE have no GPU path)" % config["model_name"])
    e, r = checkpoint_files(model_path, config["dataset"], config["model_name"])
    return config, np.load(e).astype(np.float32, copy=False), np.load(r).astype(np.float32, copy=False)


def infer_hyper(config, score_func):
    """engine.Hyper of ScoreInfer.load_model: gamma = 0 under 'none', the config's under 'logsigmoid'.  Hyper.emb_init
    = (gamma + 2) / hidden_dim then reproduces InferModel's RotatE phase scale."""
    if score_func not in ("none", "logsigmoid"):
        raise SystemExit("score function should be none or logsigmoid")
    model = "TransE_l2" if config["model_name"] == "TransE" else config["model_name"]
    gamma = float(config["gamma"]) if score_func == "logsigmoid" else 0.0
    return Hyper(model=model, hidden_dim=int(config["hidden_dim"]), gamma=gamma, double_ent=bool(config["double_ent"]),
                 double_rel=bool(config["double_rel"]))


# ------------------------------------------------------------------------------------------------------------ planning
class Plan:
    """How one exec mode maps onto score tiles, for lists of nH heads, nR relations and nT tails.
      n_lists           G, the number of result lists
      head_candidates   the H list is the candidate (column) side (batch_tail), else the T list (triplet_wise: neither)
      cstride           key step from one candidate to the next
      queries(b, e)     the queries [b, e) in tile order as (position arrays of the query sides, list, qoff): (i, j) for
                        tail candidates, (j, k) for head candidates, (i,) for triplet_wise; a list's queries are
                        consecutive
    Key of (query, candidate position c) = qoff + c * cstride."""

    def __init__(self, exec_mode, nH, nR, nT):
        if exec_mode not in EXEC_MODES:
            raise SystemExit("unknow execution mode type {}".format(exec_mode))
        self.mode, self.nH, self.nR, self.nT = exec_mode, nH, nR, nT
        self.head_candidates = exec_mode == "batch_tail"
        if exec_mode == "triplet_wise":
            if not nH == nR == nT:
                raise SystemExit("For triplet wise exection mode, head, relation and tail lists should have same length")
            self.n_queries, self.n_lists, self.cstride, self.n_cand = 1, 1, 1, nH
        elif self.head_candidates:
            self.n_queries, self.n_lists, self.cstride, self.n_cand = nR * nT, nT, nR * nT, nH
        else:
            self.n_queries, self.n_cand, self.cstride = nH * nR, nT, 1
            self.n_lists = {"all": 1, "batch_head": nH, "batch_rel": nR}[exec_mode]

    def queries(self, b, e):
        q = np.arange(b, e, dtype=np.int64)
        nH, nR, nT = self.nH, self.nR, self.nT
        if self.mode == "triplet_wise":
            return (q,), np.zeros_like(q), np.zeros_like(q)
        if self.head_candidates:                                  # k-major (k, j)
            k, j = q // nR, q % nR
            return (j, k), k, j * nT + k
        if self.mode == "batch_rel":                              # j-major (j, i)
            j, i = q // nH, q % nH
            g = j
        else:                                                     # i-major (i, j)
            i, j = q // nR, q % nR
            g = i if self.mode == "batch_head" else np.zeros_like(q)
        return (i, j), g, (i * nR + j) * nT

    def decode(self, keys):
        """Positions (i, j, k) in the H, R and T lists of keys (triplet_wise: key i is row i of all three)."""
        keys = np.asarray(keys, dtype=np.int64)
        if self.mode == "triplet_wise":
            return keys, keys, keys
        return keys // (self.nR * self.nT), (keys // self.nT) % self.nR, keys % self.nT


# ----------------------------------------------------------------------------------------------------------- execution
class Predictor:
    """Top-K link prediction over an entity and a relation table (numpy or torch, float32) on one GPU.  Runs on a library
    handle of its own, on the current stream of `device`."""

    def __init__(self, hp, ent, rel, device=0, budget=EVAL_BUDGET_BYTES, query_batch=QUERY_BATCH):
        self.hp, self.budget, self.query_batch = hp, budget, query_batch
        if hp.model not in _lib.MODEL_IDS:
            raise SystemExit("model %s is not supported by dglke_b200" % hp.model)
        self.h = _lib.Handle(device)
        self.device, self.lib = self.h.device, self.h.lib
        ent = torch.as_tensor(ent, dtype=torch.float32)
        rel = torch.as_tensor(rel, dtype=torch.float32)
        if ent.shape[1] != hp.entity_dim or rel.shape[1] != hp.relation_dim:
            raise SystemExit("table widths (%d, %d) do not match the config's model (%d, %d)"
                             % (ent.shape[1], rel.shape[1], hp.entity_dim, hp.relation_dim))
        need = (ent.numel() + rel.numel() * (2 if hp.model == "RESCAL" else 1)) * 4
        free, total = torch.cuda.mem_get_info(self.device)
        if need + 2 * budget > free:
            raise SystemExit("the tables need %.2f GB on cuda:%d, which has %.2f GB free of %.2f GB: prediction needs the "
                             "entity table on one GPU" % (need / 1e9, self.device.index, free / 1e9, total / 1e9))
        self.ent = ent.to(self.device).contiguous()
        self.rel = rel.to(self.device).contiguous()
        self.n_ent, self.n_rel = self.ent.shape[0], self.rel.shape[0]
        self._t_ent = DeviceTable.from_tensors(self.ent, torch.zeros(self.n_ent, device=self.device))
        self._t_rel = DeviceTable.from_tensors(self.rel, torch.zeros(self.n_rel, device=self.device))
        self._t_relT = None
        if hp.model == "RESCAL":                 # M_r^T, for tail candidates (module docstring)
            D = hp.entity_dim
            relT = self.rel.view(self.n_rel, -1, D).transpose(1, 2).contiguous().view(self.n_rel, -1)
            self._t_relT = DeviceTable.from_tensors(relT, torch.zeros(self.n_rel, device=self.device))

    def close(self):
        self.h.close()

    def _gather(self, table, idx):
        out = torch.empty((idx.numel(), table.dim), dtype=torch.float32, device=self.device)
        _lib.check(self.lib.kge_gather(self.h.raw, table.ref(), idx.data_ptr(), idx.numel(), out.data_ptr(),
                                       self.h.stream()))
        return out

    def tiles(self, plan, H, R, T):
        """Yields (S [Q, N] device scores, qgroup, qoff, cbase) of every tile, in order; S is reused between tiles.
        H, R, T: device id tensors (or None: every entity / relation, in id order)."""
        hp, stream = self.hp, self.h.stream()
        ar = lambda n: torch.arange(n, device=self.device)
        Hd = H if H is not None else ar(self.n_ent)
        Rd = R if R is not None else ar(self.n_rel)
        Td = T if T is not None else ar(self.n_ent)
        if plan.mode == "triplet_wise":
            row = 4 * (2 * hp.entity_dim + hp.relation_dim + 1)
            nb = max(1, min(plan.n_cand, self.budget // row))
            S = torch.empty(nb, dtype=torch.float32, device=self.device)
            zero = torch.zeros(1, dtype=torch.int64, device=self.device)
            for b in range(0, plan.n_cand, nb):
                n = min(nb, plan.n_cand - b)
                hr, rr, tr = (self._gather(t, x[b:b + n]) for t, x in ((self._t_ent, Hd), (self._t_rel, Rd), (self._t_ent, Td)))
                cfg = _cfg_for(hp, n, 1, 1, False)
                _lib.check(self.lib.kge_score_pos(self.h.raw, C.byref(cfg), hr.data_ptr(), rr.data_ptr(), tr.data_ptr(), n,
                                                  S.data_ptr(), stream))
                yield S[:n].view(1, n), zero, zero, b
            return
        cand_ids = H if plan.head_candidates else T           # None: every entity, scored in place
        rescal_t = hp.model == "RESCAL" and not plan.head_candidates
        neg_head = plan.head_candidates or rescal_t
        Qb = min(plan.n_queries, self.query_batch)
        nb = min(plan.n_cand, default_block_rows(hp.entity_dim, Qb, self.budget))
        S = torch.empty(Qb * nb, dtype=torch.float32, device=self.device)
        row_bytes = hp.entity_dim * 4
        for qb in range(0, plan.n_queries, Qb):
            qe = min(plan.n_queries, qb + Qb)
            Q = qe - qb
            (a, b), g, off = plan.queries(qb, qe)
            a, b = torch.from_numpy(a).to(self.device), torch.from_numpy(b).to(self.device)
            qgroup, qoff = torch.from_numpy(g).to(self.device), torch.from_numpy(off).to(self.device)
            if plan.head_candidates:                          # queries (r_j, t_k)
                rrows, kept = self._gather(self._t_rel, Rd[a]), self._gather(self._t_ent, Td[b])
            else:                                             # queries (h_i, r_j)
                kept = self._gather(self._t_ent, Hd[a])
                rrows = self._gather(self._t_relT if rescal_t else self._t_rel, Rd[b])
            for c0 in range(0, plan.n_cand, nb):
                n = min(nb, plan.n_cand - c0)
                if cand_ids is None:
                    blk = C.c_void_p(self.ent.data_ptr() + c0 * row_bytes)
                else:
                    crow = self._gather(self._t_ent, cand_ids[c0:c0 + n])
                    blk = C.c_void_p(crow.data_ptr())
                cfg = _cfg_for(hp, Q, Q, n, neg_head)
                heads, tails = (blk, kept.data_ptr()) if neg_head else (kept.data_ptr(), blk)
                _lib.check(self.lib.kge_score_neg(self.h.raw, C.byref(cfg), heads, rrows.data_ptr(), tails, S.data_ptr(),
                                                  stream))
                yield S[:Q * n].view(Q, n), qgroup, qoff, c0

    def topk_keys(self, plan, H, R, T, k):
        """The raw lists: (scores [G, K], keys [G, K]) as device tensors, empty slots -inf / -1."""
        K = int(k)
        if K > _lib.KGE_TOPK_MAX:
            raise SystemExit("--topK %d is above the limit of %d (KGE_TOPK_MAX)" % (K, _lib.KGE_TOPK_MAX))
        G = plan.n_lists
        top_s = torch.full((G, K), float("-inf"), dtype=torch.float32, device=self.device)
        top_k = torch.full((G, K), -1, dtype=torch.int64, device=self.device)
        stream = self.h.stream()
        for S, qgroup, qoff, cbase in self.tiles(plan, H, R, T):
            Q, N = S.shape
            _lib.check(self.lib.kge_topk(self.h.raw, S.data_ptr(), N, Q, N, qgroup.data_ptr(), qoff.data_ptr(), cbase,
                                         plan.cstride, K, G, top_s.data_ptr(), top_k.data_ptr(), stream))
        return top_s, top_k

    def topk(self, head=None, rel=None, tail=None, exec_mode="all", k=10, score_func="none"):
        """ScoreInfer.topK: [(heads, rels, tails, scores)] per list, numpy, best first (only the triples that exist)."""
        nH = self.n_ent if head is None else len(head)
        nR = self.n_rel if rel is None else len(rel)
        nT = self.n_ent if tail is None else len(tail)
        plan = Plan(exec_mode, nH, nR, nT)
        for lst, n_all, what in ((head, self.n_ent, "head"), (rel, self.n_rel, "relation"), (tail, self.n_ent, "tail")):
            if lst is not None and len(lst) and (np.min(lst) < 0 or np.max(lst) >= n_all):
                raise SystemExit("a %s id is outside [0, %d)" % (what, n_all))
        ids = [None if x is None else torch.as_tensor(np.asarray(x, dtype=np.int64)).to(self.device)
               for x in (head, rel, tail)]
        top_s, top_k = self.topk_keys(plan, *ids, k) if min(nH, nR, nT) > 0 else (
            torch.empty(plan.n_lists, 0), torch.empty(plan.n_lists, 0, dtype=torch.int64))
        top_s, top_k = top_s.cpu(), top_k.cpu().numpy()
        if score_func == "logsigmoid":
            top_s = torch.nn.functional.logsigmoid(top_s)
        top_s = top_s.numpy()
        full = lambda x, n: np.arange(n, dtype=np.int64) if x is None else np.asarray(x, dtype=np.int64)
        Hn, Rn, Tn = full(head, nH), full(rel, nR), full(tail, nT)
        out = []
        for g in range(plan.n_lists):
            m = top_k[g] >= 0
            i, j, kk = plan.decode(top_k[g][m])
            out.append((Hn[i], Rn[j], Tn[kk], top_s[g][m]))
        return out


def write_result(path, result, id2e=None, id2r=None):
    """infer_score.py's file: a header, then one line per triple, lists in order, each best first."""
    with open(path, "w+") as f:
        f.write("head\trel\ttail\tscore\n")
        for hl, rl, tl, sl in result:
            for h, r, t, s in zip(hl.tolist(), rl.tolist(), tl.tolist(), sl.tolist()):
                if id2e is not None:
                    h, r, t = id2e[h], id2r[r], id2e[t]
                f.write("{}\t{}\t{}\t{}\n".format(h, r, t, s))


def main(argv=None):
    args = ArgParser().parse_args(argv)
    if args.gpu < 0:
        raise SystemExit(NO_GPU)
    config, ent, rel = load_checkpoint(args.model_path)
    hp = infer_hyper(config, args.score_func)
    head, rel_ids, tail, (id2e, id2r) = read_lists(args.format, args.data_files, args.raw_data, args.entity_mfile,
                                                   args.rel_mfile)
    torch.cuda.set_device(args.gpu)
    p = Predictor(hp, ent, rel, args.gpu)
    try:
        result = p.topk(head, rel_ids, tail, args.exec_mode, args.topK, args.score_func)
    finally:
        p.close()
    write_result(args.output, result, id2e if args.raw_data else None, id2r if args.raw_data else None)
    print("Inference Done")
    print("The result is saved in {}".format(args.output))


if __name__ == "__main__":
    sys.exit(main())
