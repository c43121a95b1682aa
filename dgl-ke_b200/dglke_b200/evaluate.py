"""Filtered link-prediction evaluation over any DeviceTable -- one shard on one GPU, or the row-sharded entity table of
dglke_b200.dist -- with ranks counted on the GPU (reference: EvalDataset / EvalSampler, dataloader/sampler.py:538-696;
KEModel.forward_test, general_models.py:436-485; the pooled test block of train.py:330-369).

    rank = 1 + #{j : s_j >= s_pos and candidate j is not a known triple}      (IEEE >=: a NaN never counts)

Candidates
  full-entity (neg_sample_size < 0)  every entity: for each shard, blocks of at most `block_rows` rows of that shard are
                                     scored in place (kge_score_neg on the block's row pointer, a peer pointer for a remote
                                     shard), so no candidate row is gathered; kge_rank_count takes the block's first id
  sampled (neg_sample_size = N > 0)  the reference's EvalSampler with neg_chunk_size = N: positives in chunks of N, each
                                     chunk ranked against N entities drawn uniformly with replacement (seeded, per rank)
Known triples: train | valid | test, as TripleFilter; the index (FilterIndex) is two sorted (key, entity) lists, restricted
to the keys the evaluated edges use and uploaded once.  kge_rank_finish sums {1/r, r, r<=1, r<=3, r<=10, count} into a
float64 accumulator that the host reads once per evaluation."""
import ctypes as C

import numpy as np
import torch

from . import _lib
from .engine import _cfg_for

METRICS = ("MRR", "MR", "HITS@1", "HITS@3", "HITS@10")

# Block size of full-entity evaluation.  kge_score_neg's stand-alone workspace grows with the candidate rows of a block:
# 5 D floats per row for the row and its TF32 hi/lo slabs (two layouts), 4 scalars, and per query 4 [Q, rows] planes
# (scores, coefficients, their hi/lo) plus 2 of the transposed coefficient slabs padded to 32 queries; the caller's score
# tile adds one more plane.  EVAL_BUDGET_BYTES bounds that block-proportional part, so an evaluation beside a training
# run that fills the GPU asks for about 1 GiB more (the library keeps 1/4 of headroom on top).
EVAL_BUDGET_BYTES = 1 << 30


def default_block_rows(entity_dim, n_queries, budget=EVAL_BUDGET_BYTES):
    """Largest multiple of 8 rows (full blocks keep the wgmma engine) whose workspace fits the budget."""
    q32 = -(-n_queries // 32) * 32
    per_row = 4 * (5 * entity_dim + 8 + 5 * n_queries + 2 * q32)
    return max(8, (budget // per_row) // 8 * 8)


# ------------------------------------------------------------------------------------------------ host-side selection
def select_eval_edges(split, eval_percent, seed=0):
    """--eval_percent p < 1: int(n p) edges drawn with replacement (EvalDataset, sampler.py:686-696), seeded."""
    if eval_percent >= 1:
        return split
    n = len(split[0])
    idx = np.random.default_rng(seed).integers(0, n, int(n * eval_percent))
    return tuple(np.asarray(x)[idx] for x in split[:3])


def rank_slice(n, rank, world):
    """[begin, end) of the edges rank `rank` of `world` evaluates (EvalDataset.create_sampler, sampler.py:773-774)."""
    return n * rank // world, min(n * (rank + 1) // world, n)


def eval_chunks(n, batch_size, neg_sample_size):
    """[(begin, end, num_chunks, chunk_size)] of the evaluation batches of n edges.  Full-entity (neg_sample_size < 0):
    every batch is one chunk.  Sampled: chunks of neg_sample_size positives; a last batch with fewer positives is one
    chunk, a larger one that is not a multiple of it is dropped (create_neg_subgraph, sampler.py:486-512)."""
    out = []
    for s in range(0, n, batch_size):
        b = min(batch_size, n - s)
        if neg_sample_size < 0 or b < neg_sample_size:
            out.append((s, s + b, 1, b))
        elif b % neg_sample_size == 0:
            out.append((s, s + b, b // neg_sample_size, neg_sample_size))
    return out


def metrics_from_sums(sums):
    """{MRR, MR, HITS@1, HITS@3, HITS@10} of the six sums kge_rank_finish accumulates (pooled means: the sums may come
    from several ranks with slices of different sizes)."""
    sums = np.asarray(sums, dtype=np.float64)
    return {k: float(sums[i] / sums[5]) for i, k in enumerate(METRICS)} if sums[5] > 0 else {}


def check_eval_flags(args):
    """--neg_deg_sample_eval is a forward_test feature (the reference forbids it with the filter anyway, train.py:106)."""
    if getattr(args, "neg_deg_sample_eval", False) and (len(args.gpu) > 1 or args.neg_sample_size_eval > 0):
        raise ValueError("--neg_deg_sample_eval works with one GPU and full-entity ranking only "
                         "(not with several --gpu ids or --neg_sample_size_eval > 0)")


class FilterIndex:
    """The known triples as two sorted lists per corruption side: keys = kept_entity * n_rel + rel (int64) and vals = the
    corrupted side's entity (int32), sorted and distinct within each key.  'head' ranks corrupted heads (kept = tail),
    'tail' corrupted tails (kept = head)."""

    def __init__(self, sides, n_rel):
        self.sides, self.n_rel = sides, int(n_rel)

    @classmethod
    def build(cls, heads, rels, tails, n_rel):
        h, r, t = (np.asarray(a, dtype=np.int64) for a in (heads, rels, tails))

        def side(kept, corrupted):
            key = kept * n_rel + r
            o = np.lexsort((corrupted, key))
            key, val = key[o], corrupted[o]
            first = np.ones(len(key), dtype=bool)
            first[1:] = (key[1:] != key[:-1]) | (val[1:] != val[:-1])
            return key[first], val[first].astype(np.int32)
        return cls({"head": side(t, h), "tail": side(h, t)}, n_rel)

    def restrict(self, heads, rels, tails):
        """Only the keys that these query edges use (a rank then holds its own share of a large graph's filter)."""
        h, r, t = (np.asarray(a, dtype=np.int64) for a in (heads, rels, tails))
        out = {}
        for name, kept in (("head", t), ("tail", h)):
            keys, vals = self.sides[name]
            m = np.isin(keys, np.unique(kept * self.n_rel + r))
            out[name] = (keys[m], vals[m])
        return FilterIndex(out, self.n_rel)

    def known(self, name, kept, rel):
        """The known corrupted-side entities of one query (host; tests)."""
        keys, vals = self.sides[name]
        k = int(kept) * self.n_rel + int(rel)
        return vals[np.searchsorted(keys, k, "left"):np.searchsorted(keys, k, "right")]

    def upload(self, device):
        return DeviceFilter(self, device)


class DeviceFilter:
    """A FilterIndex in device memory: one kge_filter_t per side."""

    def __init__(self, index, device):
        self.keep, self.c = [], {}
        for name, (keys, vals) in index.sides.items():
            k = torch.from_numpy(np.ascontiguousarray(keys)).to(device)
            v = torch.from_numpy(np.ascontiguousarray(vals)).to(device)
            self.keep += [k, v]
            self.c[name] = _lib.Filter(k.data_ptr(), v.data_ptr(), k.numel(), index.n_rel)


class EvalSplit:
    """One split (after the --eval_percent selection) as rank `rank` of `world` evaluates it: its slice of the edges on
    the device and, for filtered evaluation, the filter index restricted to the slice's keys, uploaded."""

    def __init__(self, split, device, index=None, rank=0, world=1):
        h, r, t = split[:3]
        b, e = rank_slice(len(h), rank, world)
        h, r, t = (np.ascontiguousarray(np.asarray(x, dtype=np.int64)[b:e]) for x in (h, r, t))
        self.n = e - b
        self.heads, self.rels, self.tails = (torch.from_numpy(x).to(device) for x in (h, r, t))
        self.filter = index.restrict(h, r, t).upload(device) if index is not None else None


class Evaluator:
    """Ranks of evaluation queries over the entity table `ent` (a DeviceTable of any number of shards) and the relation
    table `rel`.  It runs on a library handle of its own, on the caller's current stream: its stand-alone workspace never
    overlays the training step's (arena, node-gradient region, rows staged by kge_set_next_batch), and the stream orders
    it after the steps before it and before the steps after it.  close() frees the workspace."""

    def __init__(self, hp, ent, rel, device, block_rows=None, seed=0):
        self.hp, self.ent, self.rel = hp, ent, rel
        self.h = _lib.Handle(device)
        self.device, self.lib = self.h.device, self.h.lib
        self.block_rows = block_rows
        self.gen = torch.Generator(device=self.device).manual_seed(seed)
        self.acc = torch.zeros(6, dtype=torch.float64, device=self.device)

    def close(self):
        self.h.close()

    def _gather(self, table, idx):
        out = torch.empty((idx.numel(), table.dim), dtype=torch.float32, device=self.device)
        _lib.check(self.lib.kge_gather(self.h.raw, table.ref(), idx.data_ptr(), idx.numel(), out.data_ptr(),
                                       self.h.stream()))
        return out

    def _score_neg(self, heads, rel, tails, out, num_chunks, chunk_size, n_cand, neg_head):
        cfg = _cfg_for(self.hp, num_chunks * chunk_size, chunk_size, n_cand, neg_head)
        _lib.check(self.lib.kge_score_neg(self.h.raw, C.byref(cfg), heads, rel, tails, out.data_ptr(), self.h.stream()))

    def _shard_blocks(self, block_rows):
        """(first id, rows, row pointer) of every block: blocks never cross a shard's end."""
        t = self.ent.ctable
        row_bytes = t.dim * 4
        for s in range(t.n_shards):
            sh = t.shards[s]
            for b0 in range(sh.row_begin, sh.row_end, block_rows):
                yield b0, min(block_rows, sh.row_end - b0), sh.emb + (b0 - sh.row_begin) * row_bytes

    def rank_batch(self, h, r, t, neg_head, filt=None, neg_sample_size=-1, num_chunks=1, want_ranks=False,
                   want_cand=False):
        """Rank one batch of queries (int64 device tensors h, r, t) against every entity (neg_sample_size < 0) or against
        neg_sample_size sampled candidates per chunk of len(h) / num_chunks queries; adds to self.acc.  Returns the
        ranks (want_ranks) and the candidate ids [num_chunks, N] (want_cand), else None."""
        hp, Q = self.hp, h.numel()
        side = "head" if neg_head else "tail"
        kept_ids = t if neg_head else h
        H, R, T = self._gather(self.ent, h), self._gather(self.rel, r), self._gather(self.ent, t)
        pos = torch.empty(Q, dtype=torch.float32, device=self.device)
        cfg = _cfg_for(hp, Q, 1, 1, False)
        stream = self.h.stream()
        _lib.check(self.lib.kge_score_pos(self.h.raw, C.byref(cfg), H.data_ptr(), R.data_ptr(), T.data_ptr(), Q,
                                          pos.data_ptr(), stream))
        kept = T if neg_head else H
        cnt = torch.zeros(Q, dtype=torch.int64, device=self.device)
        fc = C.byref(filt.c[side]) if filt is not None else None
        cand = None
        if neg_sample_size < 0:
            nb = self.block_rows or default_block_rows(hp.entity_dim, Q)
            S = torch.empty(Q * min(nb, self.ent.num_rows), dtype=torch.float32, device=self.device)
            for base, rows, ptr in self._shard_blocks(nb):
                blk = C.c_void_p(ptr)
                self._score_neg(blk if neg_head else kept.data_ptr(), R.data_ptr(), kept.data_ptr() if neg_head else blk,
                                S, 1, Q, rows, neg_head)
                _lib.check(self.lib.kge_rank_count(self.h.raw, S.data_ptr(), rows, Q, rows, pos.data_ptr(), base, None, Q,
                                                   kept_ids.data_ptr(), r.data_ptr(), fc, cnt.data_ptr(), stream))
        else:
            N, Cs = neg_sample_size, Q // num_chunks
            cand = torch.randint(0, self.ent.num_rows, (num_chunks, N), generator=self.gen, device=self.device)
            rows = self._gather(self.ent, cand.view(-1))
            S = torch.empty(Q * N, dtype=torch.float32, device=self.device)
            self._score_neg(rows.data_ptr() if neg_head else kept.data_ptr(), R.data_ptr(),
                            kept.data_ptr() if neg_head else rows.data_ptr(), S, num_chunks, Cs, N, neg_head)
            _lib.check(self.lib.kge_rank_count(self.h.raw, S.data_ptr(), N, Q, N, pos.data_ptr(), 0, cand.data_ptr(), Cs,
                                               kept_ids.data_ptr(), r.data_ptr(), fc, cnt.data_ptr(), stream))
        ranks = torch.empty(Q, dtype=torch.int64, device=self.device) if want_ranks else None
        _lib.check(self.lib.kge_rank_finish(self.h.raw, cnt.data_ptr(), Q, ranks.data_ptr() if want_ranks else None,
                                            self.acc.data_ptr(), stream))
        if want_cand:
            return ranks, cand
        return ranks

    def run(self, split, batch_size, neg_sample_size=-1):
        """Both corruption sides of an EvalSplit (heads first, as the reference's sampler list); returns the six sums
        as a float64 device tensor [6] (self.acc, zeroed first)."""
        self.acc.zero_()
        for neg_head in (True, False):
            for b, e, nc, _ in eval_chunks(split.n, batch_size, neg_sample_size):
                self.rank_batch(split.heads[b:e], split.rels[b:e], split.tails[b:e], neg_head, split.filter,
                                neg_sample_size, nc)
        return self.acc
