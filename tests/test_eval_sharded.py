"""Host side of the GPU-counted evaluation (dglke_b200.evaluate): the filter index, the --eval_percent selection and the
per-rank slices, the sampled-mode chunking, the pooling of per-rank sums, and the refused flag combinations."""
import os
import re

import numpy as np
import pytest

from dglke_b200 import evaluate as ev
from dglke_b200.graph import TripleFilter
from dglke_b200.utils import ArgParser


def _graph_with_hubs(n_ent, n_rel, n, seed):
    """Random triples plus a (head, rel) with many tails, a (tail, rel) with many heads, and duplicated triples."""
    rng = np.random.default_rng(seed)
    h, r, t = rng.integers(0, n_ent, n), rng.integers(0, n_rel, n), rng.integers(0, n_ent, n)
    hub_t = rng.integers(0, n_ent, 400)
    hub_h = rng.integers(0, n_ent, 400)
    h = np.concatenate([h, np.full(400, 7), hub_h, h[:50]])
    r = np.concatenate([r, np.full(400, 1), np.full(400, 2), r[:50]])
    t = np.concatenate([t, hub_t, np.full(400, 11), t[:50]])
    return h, r, t


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_filter_index_excludes_what_triple_filter_biases(seed):
    n_ent, n_rel = 503, 5
    h, r, t = _graph_with_hubs(n_ent, n_rel, 3000, seed)
    rng = np.random.default_rng(seed + 10)
    q = np.concatenate([rng.integers(0, len(h), 200), [3000, 3400]])      # queries include both hub keys
    qh, qr, qt = h[q], r[q], t[q]
    tf = TripleFilter(h, r, t, n_rel)
    full = ev.FilterIndex.build(h, r, t, n_rel)
    restricted = full.restrict(qh, qr, qt)
    for neg_head, side in ((True, "head"), (False, "tail")):
        bias = tf.bias(qh, qr, qt, n_ent, neg_head)
        for idx in (full, restricted):
            keys, vals = idx.sides[side]
            assert np.all(np.diff(keys) >= 0)
            for i in range(len(q)):
                got = idx.known(side, qt[i] if neg_head else qh[i], qr[i])
                assert np.all(np.diff(got) > 0), "vals must be sorted and distinct within a key"
                assert got.tolist() == np.nonzero(bias[i] == -1)[0].tolist()
        # the restricted index holds only keys the queries use
        used = set(((qt if neg_head else qh) * n_rel + qr).tolist())
        assert set(restricted.sides[side][0].tolist()) <= used
    assert len(full.known("tail", 7, 1)) > 200 and len(full.known("head", 11, 2)) > 200


@pytest.mark.parametrize("n,p,world", [(1000, 0.5, 2), (997, 0.3, 3), (59071, 0.1, 8), (10, 1.0, 3), (5, 1.0, 8)])
def test_eval_percent_selection_and_rank_slices_cover_each_chosen_edge_once(n, p, world):
    split = (np.arange(n), np.arange(n) % 7, np.arange(n) * 3)
    sel = ev.select_eval_edges(split, p, seed=4)
    m = len(sel[0])
    assert m == (int(n * p) if p < 1 else n)
    if p < 1:
        assert sel[0].tolist() == np.random.default_rng(4).integers(0, n, int(n * p)).tolist()   # with replacement
    else:
        assert sel is split
    seen = np.zeros(m, dtype=int)
    prev_end = 0
    for r in range(world):
        b, e = ev.rank_slice(m, r, world)
        assert b == prev_end and e >= b
        seen[b:e] += 1
        prev_end = e
    assert prev_end == m and (seen == 1).all()


def test_sampled_chunking_follows_the_last_batch_rules():
    # batch_size_eval made compatible with N = 8: multiple of 8
    assert ev.eval_chunks(40, 16, 8) == [(0, 16, 2, 8), (16, 32, 2, 8), (32, 40, 1, 8)]
    assert ev.eval_chunks(37, 16, 8) == [(0, 16, 2, 8), (16, 32, 2, 8), (32, 37, 1, 5)]   # fewer than N: one chunk
    assert ev.eval_chunks(45, 24, 8) == [(0, 24, 3, 8)]                                     # 21 % 8 != 0: dropped
    assert ev.eval_chunks(30, 8, 1000) == [(0, 8, 1, 8), (8, 16, 1, 8), (16, 24, 1, 8), (24, 30, 1, 6)]
    # full-entity: one chunk per batch, the last one included
    assert ev.eval_chunks(35, 16, -1) == [(0, 16, 1, 16), (16, 32, 1, 16), (32, 35, 1, 3)]


def test_pooled_means_from_unequal_rank_slices():
    rng = np.random.default_rng(0)
    ranks = rng.integers(1, 50, 1001)
    sums = []
    for r in range(3):
        b, e = ev.rank_slice(len(ranks), r, 3)
        x = ranks[b:e].astype(np.float64)
        sums.append(np.array([(1 / x).sum(), x.sum(), (x <= 1).sum(), (x <= 3).sum(), (x <= 10).sum(), len(x)]))
    pooled = ev.metrics_from_sums(np.sum(sums, 0))
    x = ranks.astype(np.float64)
    want = {"MRR": (1 / x).mean(), "MR": x.mean(), "HITS@1": (x <= 1).mean(), "HITS@3": (x <= 3).mean(),
            "HITS@10": (x <= 10).mean()}
    for k, v in want.items():
        assert abs(pooled[k] - v) <= 1e-12 * abs(v), k
    # slices of 333, 334 and 334 ranks: the mean of the per-rank means is not the pooled mean
    per_rank = np.mean([ev.metrics_from_sums(s)["MR"] for s in sums])
    assert [int(s[5]) for s in sums] == [333, 334, 334] and per_rank != pooled["MR"]


@pytest.mark.parametrize("argv", [["--gpu", "0", "1", "--neg_deg_sample_eval"],
                                  ["--gpu", "0", "--neg_deg_sample_eval", "--neg_sample_size_eval", "100"]])
def test_refused_flag_combinations(argv):
    with pytest.raises(ValueError, match="neg_deg_sample_eval"):
        ev.check_eval_flags(ArgParser().parse_args(argv))
    from dglke_b200 import train
    with pytest.raises(ValueError, match="neg_deg_sample_eval"):
        train.main(argv)


def test_accepted_flag_combinations():
    for argv in (["--gpu", "0", "--neg_deg_sample_eval"], ["--gpu", "0", "1", "--neg_sample_size_eval", "100"]):
        ev.check_eval_flags(ArgParser().parse_args(argv))


def test_default_block_rows_is_a_multiple_of_8_within_the_budget():
    for d, q in ((400, 16), (400, 1000), (800, 8), (64, 3)):
        nb = ev.default_block_rows(d, q)
        assert nb % 8 == 0 and nb >= 8
        q32 = -(-q // 32) * 32
        assert nb * 4 * (5 * d + 8 + 5 * q + 2 * q32) <= ev.EVAL_BUDGET_BYTES
    assert ev.default_block_rows(400, 16) >= 14952          # FB15k: one block at the usual eval batch


LOG = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "dgl-ke_b200", "build",
                   "kge_eval.ptxas.log")


@pytest.mark.skipif(not os.path.exists(LOG), reason="no compiler log: the library was not built here")
@pytest.mark.parametrize("kernel", ["_ZN3kge12k_rank_countE", "_ZN3kge13k_rank_finishE"])
def test_rank_kernel_does_not_spill(kernel):
    """k_rank_count: 32 registers, k_rank_finish: 40 (CUDA 12.9, sm_90a)."""
    blocks = re.split(r"ptxas info\s+: Compiling entry function ", open(LOG).read())
    hit = [b for b in blocks if b.startswith("'") and b.split("'")[1].startswith(kernel)]
    assert len(hit) == 1, "no compiler output for %s" % kernel
    assert "0 bytes spill stores, 0 bytes spill loads" in hit[0].split("Used")[0], hit[0][:400]
