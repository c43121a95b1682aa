"""Evaluation with ranks counted on the GPU (dglke_b200.evaluate: kge_score_neg tiles -> kge_rank_count ->
kge_rank_finish) over one-shard and sharded entity tables.

Ranks are checked against the float64 near-tie intervals of test_gpu_eval_scores.py (the truth computed from the rows,
not from the device's scores), against forward_test's ranks where both see the same score tile, and exactly where the
filter holds hub keys.  Sharded tables are those of test_gpu_sharded.py: one allocation per shard with NaN rows past its
end, so a block that crosses a shard's end reads NaN scores, which never count, and shows up as a wrong rank."""
import os

import numpy as np
import pytest
import torch as th

from test_gpu_eval_scores import (N_REL, TILE, _hypers, _known_triples, _planted, _rank_intervals, _score_routes,
                                  _seed, _tables, _filter_mask)
from test_gpu_plugin import _args
from test_gpu_sharded import (PF_SHAPES, TOL, _batch, _deferred, _engine, _hyper, _init, _on_device, _pool,
                              _sharded_step, sharded)  # noqa: F401  (sharded: fixture)

pytestmark = pytest.mark.gpu

DEV = th.device("cuda", 0)
MODELS = [("TransE_l1", 200), ("TransE_l2", 400), ("DistMult", 400), ("ComplEx", 200), ("RESCAL", 32), ("RotatE", 100)]
# (name, entities, candidates per chunk (-1: all), queries, batch_size_eval)
CASES = [("full14951", 14951, -1, 61, 16), ("full14952", 14952, -1, 61, 16), ("sampled1000", 1500, 1000, 2203, 2000)]
SMALL_BLOCK = 2501              # unaligned: ragged blocks, filtered sets straddling block boundaries


def _setup(khp, n_ent, n_test, seed):
    """Tables and query triples: planted near the top for TransE_l2 / DistMult, 'trained-like' random otherwise."""
    if khp.model in ("TransE_l2", "DistMult"):
        ent, rel, (H, R, T), _ = _planted(khp, n_ent, n_test, seed)
        return ent, rel, H, R, T
    ent, rel = _tables(khp, n_ent, N_REL, "trained", seed)
    rng = np.random.default_rng(seed)
    return ent, rel, rng.integers(0, n_ent, n_test), rng.integers(0, N_REL, n_test), rng.integers(0, n_ent, n_test)


def _route(model, Q, rows):
    if model in ("TransE_l1", "RotatE"):
        return TILE["l1" if model == "TransE_l1" else "rot"]
    if model == "RESCAL":
        return TILE["dot"]
    return "wgmma" if Q % 8 == 0 and rows % 8 == 0 else TILE["dot"]


def _blocks(n_ent, n_shards, block_rows):
    per = -(-n_ent // n_shards)
    out = []
    for s in range(n_shards):
        lo, hi = s * per, min(n_ent, (s + 1) * per)
        out += [min(block_rows, hi - b) for b in range(lo, hi, block_rows)]
    return out


def _rel_table(rel):
    from dglke_b200.engine import DeviceTable
    r = rel.to(DEV).contiguous()
    return DeviceTable.from_tensors(r, th.zeros(r.shape[0], device=DEV))


def _check_sums(acc, ranks, what):
    """kge_rank_finish's accumulator against the returned ranks: exact for MR, HITS and the count, 1e-12 for MRR."""
    x = th.cat(ranks).cpu().double()
    got = acc.cpu()
    want = [(1 / x).sum(), x.sum(), (x <= 1).sum(), (x <= 3).sum(), (x <= 10).sum(), float(len(x))]
    assert abs(float(got[0]) - float(want[0])) <= 1e-12 * float(want[0]), (what, "MRR", float(got[0]), float(want[0]))
    for i in range(1, 6):
        assert float(got[i]) == float(want[i]), (what, i, float(got[i]), float(want[i]))


@pytest.mark.parametrize("case", CASES, ids=lambda c: c[0])
@pytest.mark.parametrize("model,hidden", MODELS, ids=[m for m, _ in MODELS])
def test_ranks_within_near_tie_intervals(model, hidden, case, sharded):
    from dglke_b200.evaluate import Evaluator, FilterIndex, default_block_rows, eval_chunks
    name, n_ent, N, n_test, batch = case
    khp, ehp = _hypers(model, hidden)
    seed = _seed("eval_sharded", model, name)
    ent, rel, H, R, T = _setup(khp, n_ent, n_test, seed)
    kh, kr, kt = _known_triples(H, R, T, n_ent, seed + 2)
    dfilt = FilterIndex.build(kh, kr, kt, N_REL).restrict(H, R, T).upload(DEV)
    rel_tab = _rel_table(rel)
    h_d, r_d, t_d = (th.from_numpy(np.asarray(x, dtype=np.int64)).to(DEV) for x in (H, R, T))
    truth, dup_known = {}, 0
    configs = [(k, b) for k in (1, 2, 3) for b in ((None, SMALL_BLOCK) if N < 0 else (None,))]
    for n_shards, block_rows in configs:
        tab = sharded(ent, th.zeros(n_ent), n_shards)
        for filtered in (False, True):
            ev = Evaluator(ehp, tab.table, rel_tab, DEV, block_rows=block_rows, seed=7)
            try:
                ranks = []
                for neg_head in (True, False):
                    for b, e, nc, cs in eval_chunks(n_test, batch, N):
                        ev.h.profile_enable(True)
                        rk, cand = ev.rank_batch(h_d[b:e], r_d[b:e], t_d[b:e], neg_head, dfilt if filtered else None,
                                                 N, nc, want_ranks=True, want_cand=True)
                        routes = _score_routes(ev.h)
                        ev.h.profile_enable(False)
                        nb = block_rows or default_block_rows(khp.entity_dim, e - b)
                        want_routes = {_route(model, e - b, rows) for rows in _blocks(n_ent, n_shards, nb)} if N < 0 \
                            else {_route(model, cs, N)}
                        assert routes == want_routes, (name, n_shards, block_rows, sorted(routes), sorted(want_routes))
                        ranks.append(rk)
                        got = rk.cpu()
                        for c in range(nc):
                            q0, q1 = b + c * cs, b + (c + 1) * cs
                            cands = np.arange(n_ent) if N < 0 else cand[c].cpu().numpy()
                            key = (neg_head, filtered, q0 if N > 0 else 0)
                            if key not in truth or not np.array_equal(truth[key][0], cands):
                                qs = slice(0, n_test) if N < 0 else slice(q0, q1)
                                mask = None
                                if filtered:
                                    u, inv = np.unique(cands, return_inverse=True)
                                    mask = _filter_mask(kh, kr, kt, H[qs], R[qs], T[qs], u, neg_head)[:, th.from_numpy(inv)]
                                    if N > 0:   # a known entity drawn more than once
                                        dup_known += int((mask.sum(1) > th.from_numpy(
                                            np.array([len(set(cands[mask[i].numpy()])) for i in range(mask.shape[0])]))).sum())
                                lo, hi = _rank_intervals(khp, ent, rel, H[qs], R[qs], T[qs], cands, neg_head, mask)
                                truth[key] = (cands, lo, hi, qs.start)
                            _, lo, hi, off = truth[key]
                            g = got[c * cs:(c + 1) * cs]
                            lo_c, hi_c = lo[q0 - off:q1 - off], hi[q0 - off:q1 - off]
                            bad = ((g < lo_c) | (g > hi_c)).nonzero().view(-1).tolist()
                            assert not bad, "%s %s shards=%d block_rows=%s %s neg_head=%s: ranks %s outside %s" % (
                                model, name, n_shards, block_rows, "filtered" if filtered else "raw", neg_head,
                                g[bad[:6]].tolist(), list(zip(lo_c[bad[:6]].tolist(), hi_c[bad[:6]].tolist())))
                _check_sums(ev.acc, ranks, (model, name, n_shards, block_rows, filtered))
            finally:
                ev.close()
    if N > 0:
        assert dup_known > 0, "no query saw a known entity drawn twice: the sampled case is blind to duplicates"


@pytest.mark.parametrize("model,n_ent", [("TransE_l2", 14951), ("TransE_l2", 14952), ("DistMult", 14951),
                                         ("DistMult", 14952)])
def test_ranks_equal_forward_test_with_one_block(model, n_ent):
    """One GPU, one block covering every entity: the same score tile as forward_test, so the same integers."""
    from dglke_b200.evaluate import Evaluator, FilterIndex, eval_chunks
    from dglke_b200.general_models import KEModel
    from dglke_b200.graph import TripleFilter, eval_batches
    khp, _ = _hypers(model, 400)
    seed = _seed("ft_identity", model, n_ent)
    ent, rel, (H, R, T), _ = _planted(khp, n_ent, 203, seed)
    m = KEModel(_args(eval_filter=True), model, n_ent, N_REL, 400, khp.gamma)
    m.entity_emb.emb.copy_(ent)
    m.relation_emb.emb.copy_(rel)
    kh, kr, kt = _known_triples(H, R, T, n_ent, seed + 2)
    known = TripleFilter(kh, kr, kt, N_REL)
    dfilt = FilterIndex.build(kh, kr, kt, N_REL).restrict(H, R, T).upload(DEV)
    h_d, r_d, t_d = (th.from_numpy(np.asarray(x, dtype=np.int64)).to(DEV) for x in (H, R, T))
    ev = Evaluator(m.hyper, m.entity_emb.table(), m.relation_emb.table(), DEV, block_rows=n_ent)
    try:
        for neg_head in (True, False):
            logs = []
            with th.no_grad():
                for pg, ng in eval_batches(H, R, T, n_ent, 16, neg_head, known=known):
                    m.forward_test(pg, ng, logs, 0)
            want = [int(l["MR"]) for l in logs]
            got = th.cat([ev.rank_batch(h_d[b:e], r_d[b:e], t_d[b:e], neg_head, dfilt, want_ranks=True)
                          for b, e, _, _ in eval_chunks(203, 16, -1)]).tolist()
            assert got == want, (model, n_ent, neg_head, [(i, a, b) for i, (a, b) in enumerate(zip(got, want)) if a != b][:8])
    finally:
        ev.close()


def test_hub_keys_give_exact_ranks(sharded):
    """One (h, r) with 5 000 known tails and one (t, r) whose known heads are every entity but 3, on one shard (one block)
    and on two shards in blocks of 1 496 rows: ranks equal the dense count over the same kernel's score tile."""
    from dglke_b200 import engine as E
    from dglke_b200.evaluate import Evaluator, FilterIndex
    from dglke_b200.graph import TripleFilter
    n_ent, model = 14960, "TransE_l2"
    khp, ehp = _hypers(model, 400)
    ent, rel = _tables(khp, n_ent, N_REL, "trained", _seed("hubs"))
    rng = np.random.default_rng(5)
    tails5k = rng.choice(n_ent, 5000, replace=False)
    heads_all = np.setdiff1d(np.arange(n_ent), [11, 5000, 14959])
    kh = np.concatenate([np.full(5000, 7), heads_all, rng.integers(0, n_ent, 500)])
    kr = np.concatenate([np.full(5000, 1), np.full(len(heads_all), 2), rng.integers(0, N_REL, 500)])
    kt = np.concatenate([tails5k, np.full(len(heads_all), 9), rng.integers(0, n_ent, 500)])
    # 16 queries per hub: corrupting tails of (7, 1, .) and heads of (., 2, 9), each positive a known triple
    H = np.concatenate([np.full(16, 7), heads_all[rng.choice(len(heads_all), 16)]])
    R = np.concatenate([np.full(16, 1), np.full(16, 2)])
    T = np.concatenate([tails5k[:16], np.full(16, 9)])
    tf = TripleFilter(kh, kr, kt, N_REL)
    dfilt = FilterIndex.build(kh, kr, kt, N_REL).restrict(H, R, T).upload(DEV)
    rel_d = rel.to(DEV)
    e_d = ent.to(DEV)
    for sl, neg_head in ((slice(0, 16), False), (slice(16, 32), True)):
        h, r, t = H[sl], R[sl], T[sl]
        hr, rr, tr = e_d[th.from_numpy(h)], rel_d[th.from_numpy(r)], e_d[th.from_numpy(t)]
        pos = E.score_pos(ehp, hr, rr, tr)
        S = E.score_neg(ehp, *((e_d, rr, tr) if neg_head else (hr, rr, e_d)), 1, 16, n_ent, neg_head)[0]
        bias = th.from_numpy(tf.bias(h, r, t, n_ent, neg_head)).to(DEV)
        want = (1 + ((S >= pos[:, None]) & (bias != -1)).sum(1)).tolist()
        if neg_head:
            assert max(want) <= 4
        for n_shards, block_rows in ((1, None), (2, 1496)):
            tab = sharded(ent, th.zeros(n_ent), n_shards)
            ev = Evaluator(ehp, tab.table, _rel_table(rel), DEV, block_rows=block_rows)
            try:
                d = lambda a: th.from_numpy(np.asarray(a, dtype=np.int64)).to(DEV)
                got = ev.rank_batch(d(h), d(r), d(t), neg_head, dfilt, want_ranks=True).tolist()
            finally:
                ev.close()
            assert got == want, (n_shards, neg_head, got, want)


def test_training_resumes_after_an_evaluation_with_staged_rows(sharded):
    """2-shard table, pipelined steps (step s announces step s+1, kge_set_next_batch), an evaluation between steps 0
    and 1 and between 1 and 2: the tables after step 3 match the same run without the evaluations, and the announced
    steps ran from the staged rows (one launch fewer than a step that gathers its own)."""
    from dglke_b200.evaluate import EvalSplit, Evaluator, FilterIndex
    cfg = PF_SHAPES[0]
    hp = _hyper(cfg, reg_coef=1e-4)
    n_ent, n_rel, B, Cs, Ns = cfg[5:10]
    ent, es, rel, rs = _init(hp, n_ent, n_rel)
    steps = 4
    announced = [0 < s < steps - 1 for s in range(steps)]
    rng = np.random.default_rng(3)
    va = (rng.integers(0, n_ent, 40), rng.integers(0, n_rel, 40), rng.integers(0, n_ent, 40))
    results = []
    for with_eval in (True, False):
        tab = sharded(ent, es, 2)
        eng, r, r_s = _engine(hp, tab, rel, rs)
        rg, rgs = _deferred(eng, n_rel, hp.relation_dim)
        pool = _pool(tab, n_ent, 5)
        dev = [_on_device(_batch(n_ent, n_rel, B, Cs, Ns, tab.boundary_ids(), 300 + s, s % 2 == 1, pool=pool)[0])
               for s in range(steps)]
        split = EvalSplit(va, DEV, FilterIndex.build(*va, n_rel))
        launches, sums = [], []
        for s in range(steps):
            nxt = (dev[s + 1]["node_ids"], dev[s + 1]["neg_ids"]) if s + 1 < steps and announced[s + 1] else None
            _, n = _sharded_step(eng, rg, rgs, dev[s], Cs, Ns, next_batch=nxt)
            launches.append(n)
            if with_eval and s < 2:
                ev = Evaluator(eng.hp, eng.ent, eng.rel, DEV)
                try:
                    sums.append(ev.run(split, 16).cpu())
                finally:
                    ev.close()
        th.cuda.synchronize()
        assert all(launches[s] == launches[-1] - 1 for s in range(steps) if announced[s]), \
            "staged rows were not used: launches per step %r" % (launches,)
        if with_eval:
            assert all(float(x[5]) == 80 for x in sums)
        e, st = tab.read()
        results.append((e.numpy(), st.numpy(), r.cpu().numpy(), r_s.cpu().numpy(), launches))
    (a, b) = results
    assert a[4] == b[4], (a[4], b[4])
    for x, y, what in zip(a[:4], b[:4], ("entity table", "entity state", "relation table", "relation state")):
        np.testing.assert_allclose(x, y, rtol=TOL, atol=1e-6, err_msg=what)


def test_two_ranks_pooled_evaluation():
    """tests/dist_eval_check.py under torchrun: 2 GPUs over NCCL, or both ranks on cuda:0 over gloo."""
    from test_dist import _torchrun, ROOT
    env = {} if th.cuda.device_count() >= 2 else {"DIST_SAME_GPU": "1"}
    out = _torchrun(2, os.path.join(ROOT, "tests", "dist_eval_check.py"), env=env)
    assert "DIST_EVAL_OK" in out.stdout, out.stdout[-3000:] + out.stderr[-4000:]


def _udd_argv(tmp_path, *extra):
    fx = os.path.join(os.path.dirname(os.path.abspath(__file__)), "fixtures", "udd")
    return ["--model_name", "DistMult", "--dataset", "tiny", "--format", "udd_hrt", "--data_path", fx,
            "--data_files", "entities.dict", "relations.dict", "train.txt", "valid.txt", "test.txt",
            "--batch_size", "16", "--neg_sample_size", "4", "--hidden_dim", "8", "--max_step", "20",
            "--log_interval", "10", "--save_path", str(tmp_path), "-adv", "--batch_size_eval", "4", "--lr", "0.1",
            "--neg_sample_size_eval", "8", "--eval_percent", "0.5", "--test", "--valid", "--eval_interval", "10",
            "--no_save_emb", *extra]


def test_cli_sampled_evaluation_one_gpu(tmp_path, capfd):
    from dglke_b200 import train
    train.main(_udd_argv(tmp_path, "--gpu", "0"))
    out = capfd.readouterr().out
    for k in ("MRR", "MR", "HITS@1", "HITS@3", "HITS@10"):
        assert "[0]Test average %s: " % k in out and "[0]Valid average %s: " % k in out, out[-2000:]


@pytest.mark.skipif(th.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_cli_sampled_evaluation_two_gpus(tmp_path, capfd):
    from dglke_b200 import train
    train.main(_udd_argv(tmp_path, "--gpu", "0", "1"))
    out = capfd.readouterr().out
    assert "-------------- Test result --------------" in out, out[-2000:]
    for k in ("MRR", "MR", "HITS@1", "HITS@3", "HITS@10"):
        assert "Test average %s : " % k in out and "[1]Valid average %s: " % k in out, out[-2000:]


@pytest.mark.parametrize("explicit", [False, True], ids=["range_ids", "explicit_ids"])
def test_rank_count_on_a_crafted_tile(explicit):
    """kge_rank_count / kge_rank_finish on a tile with exact ties (they count), NaN scores and a NaN positive (they
    never count), a ragged last segment, and known ids that repeat among explicit candidates (every copy excluded)."""
    import ctypes as C
    from dglke_b200 import _lib
    from dglke_b200.evaluate import FilterIndex
    rng = np.random.default_rng(11)
    Q, N, ld, base, n_rel, chunk = 24, 3000, 3011, 500, 3, 8
    S = rng.normal(size=(Q, ld)).astype(np.float32)
    pos = rng.normal(size=Q).astype(np.float32)
    S[:, :N:7] = pos[:, None]                           # exact ties
    S[:, 5:N:11] = np.nan
    pos[3] = np.nan
    kept, rel = rng.integers(0, 50, Q), rng.integers(0, n_rel, Q)
    cand = rng.integers(base, base + 400, (Q // chunk, N)) if explicit else None
    ids = cand[np.arange(Q) // chunk] if explicit else np.broadcast_to(base + np.arange(N), (Q, N))
    kh, kr, kt = [], [], []
    for q in range(Q):                                  # known tails: some inside the tile's ids, some outside
        k = rng.choice(np.arange(base - 100, base + N + 100), 300, replace=False)
        kh += [kept[q]] * len(k)
        kr += [rel[q]] * len(k)
        kt += list(k)
    dfilt = FilterIndex.build(np.array(kh), np.array(kr), np.array(kt), n_rel).upload(DEV)
    known = np.zeros((Q, N), dtype=bool)
    for q in range(Q):
        known[q] = np.isin(ids[q], np.array(kt)[(np.array(kh) == kept[q]) & (np.array(kr) == rel[q])])
    hit = S[:, :N] >= pos[:, None]
    h = _lib.Handle(0)
    try:
        for filtered in (False, True):
            want = 1 + (hit & ~known).sum(1) if filtered else 1 + hit.sum(1)
            d = lambda a, dt=th.int64: th.from_numpy(np.ascontiguousarray(a)).to(DEV, dt)
            cnt = th.zeros(Q, dtype=th.int64, device=DEV)
            acc = th.zeros(6, dtype=th.float64, device=DEV)
            ranks = th.empty(Q, dtype=th.int64, device=DEV)
            S_d, pos_d, kept_d, rel_d = d(S, th.float32), d(pos, th.float32), d(kept), d(rel)
            cand_d = d(cand) if explicit else None
            _lib.check(h.lib.kge_rank_count(h.raw, S_d.data_ptr(), ld, Q, N, pos_d.data_ptr(), 0 if explicit else base,
                                            cand_d.data_ptr() if explicit else None, chunk, kept_d.data_ptr(),
                                            rel_d.data_ptr(), C.byref(dfilt.c["tail"]) if filtered else None,
                                            cnt.data_ptr(), h.stream()))
            _lib.check(h.lib.kge_rank_finish(h.raw, cnt.data_ptr(), Q, ranks.data_ptr(), acc.data_ptr(), h.stream()))
            got = ranks.cpu().numpy()
            assert got.tolist() == want.tolist(), (filtered, [(q, a, b) for q, (a, b) in enumerate(zip(got, want)) if a != b])
            assert got[3] == 1
            _check_sums(acc, [ranks], ("crafted", explicit, filtered))
    finally:
        h.close()
