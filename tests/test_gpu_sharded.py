"""The sharded-table paths of the step (entity table split into row-range shards, as dglke_b200.dist lays it out over
several GPUs), driven in one process on cuda:0 against the CPU oracle at the hot shapes.

A table of several shards needs neither several GPUs nor several processes: kge_table_t takes up to 8 shard pointers,
and any CUDA allocations will do.  Every shard here is its own allocation, so a kernel that ignores the shard index
reads the wrong memory instead of the right row by accident, and every shard has PAD rows (and state entries) past its
end filled with NaN: a read past a shard's end shows up as NaN in the result, a write past it as changed padding, which
the `sharded` fixture checks after every test.  The boundary ids of every shard are in the heads, tails and negatives of
every batch.

Every test runs on a handle of its own: the deferred relation mode, the relation buffers and the prefetch state live on
the handle, and the rest of the suite shares get_handle(0).  Tolerances and the float64 arbitration are those of
tests/test_gpu_parity.py."""
import dataclasses

import numpy as np
import pytest
import torch as th

import kge_oracle as ko
from test_gpu_parity import _check_step

pytestmark = pytest.mark.gpu

PAD = 3
TOL = 5e-5                   # test_gpu_parity's hot-shape tolerance
FUSED_KEYS = ("log", "e", "es", "r", "rs")


class ShardedTable:
    """emb [n, D] / state [n] (CPU) split over `n_shards` row ranges of ceil(n / n_shards) rows, one allocation per shard
    on cuda:0 with PAD NaN rows and state entries behind the rows the table sees."""

    def __init__(self, emb, state, n_shards):
        from dglke_b200.engine import DeviceTable
        dev = th.device("cuda", 0)
        n, D = emb.shape
        self.per = (n + n_shards - 1) // n_shards
        self.allocs, views_e, views_s = [], [], []
        for s in range(n_shards):
            lo, hi = s * self.per, min(n, (s + 1) * self.per)
            e = th.full((hi - lo + PAD, D), float("nan"), device=dev)
            st = th.full((hi - lo + PAD,), float("nan"), device=dev)
            e[:hi - lo] = emb[lo:hi].to(dev)
            st[:hi - lo] = state[lo:hi].to(dev)
            self.allocs.append((e, st, hi - lo))
            views_e.append(e[:hi - lo])
            views_s.append(st[:hi - lo])
        self.pad_bits = [(e[r:].view(th.int32).cpu(), st[r:].view(th.int32).cpu()) for e, st, r in self.allocs]
        self.table = DeviceTable(views_e, views_s, n, D, devices=[0] * n_shards)

    def read(self):
        """(emb, state) of the whole table as CPU tensors"""
        return (th.cat([e[:r] for e, _, r in self.allocs]).cpu(), th.cat([st[:r] for _, st, r in self.allocs]).cpu())

    def boundary_ids(self):
        n = self.table.num_rows
        ids = {0, n - 1}
        for k in range(1, len(self.allocs)):
            ids |= {k * self.per - 1, k * self.per}
        return np.array(sorted(ids), dtype=np.int64)

    def check_padding(self):
        for s, ((e, st, r), (be, bs)) in enumerate(zip(self.allocs, self.pad_bits)):
            assert bool(th.isnan(e[r:]).all()) and th.equal(e[r:].view(th.int32).cpu(), be), \
                "shard %d: a row past its end was written" % s
            assert bool(th.isnan(st[r:]).all()) and th.equal(st[r:].view(th.int32).cpu(), bs), \
                "shard %d: a state entry past its end was written" % s


@pytest.fixture
def sharded():
    made = []

    def make(emb, state, n_shards):
        made.append(ShardedTable(emb, state, n_shards))
        return made[-1]
    yield make
    th.cuda.synchronize()
    for t in made:
        t.check_padding()


def _handle():
    from dglke_b200 import _lib
    return _lib.Handle(0)


def _engine(hp, tab, rel, rel_state):
    """StepEngine on a private handle over the sharded entity table and a one-allocation relation table."""
    from dglke_b200.engine import StepEngine, DeviceTable, Hyper
    r, rs = rel.cuda().contiguous(), rel_state.cuda().contiguous()
    eng = StepEngine(Hyper(**dataclasses.asdict(hp)), tab.table, DeviceTable.from_tensors(r, rs), 0)
    eng.h = _handle()
    return eng, r, rs


def _deferred(eng, n_rel, Dr):
    """ShardedTrainer's relation set-up: deferred mode, the fused step sums into caller-owned buffers."""
    from dglke_b200 import _lib
    rbuf = th.zeros(n_rel * Dr + n_rel, dtype=th.float32, device=eng.device)
    rg, rgs = rbuf[:n_rel * Dr], rbuf[n_rel * Dr:]
    _lib.check(eng.lib.kge_set_relation_mode(eng.h.raw, 1))
    _lib.check(eng.lib.kge_set_relation_buffers(eng.h.raw, rg.data_ptr(), rgs.data_ptr()))
    return rg, rgs


def _sharded_step(eng, rg, rgs, batch, Cs, Ns, next_batch=None):
    """ShardedTrainer.step with one rank (its all-reduce is the identity): begin, end, apply the relation sums.
    `batch`: a step-input dict (CUDA tensors) or a DeviceBatch.  Returns (log4 on the host, kernels launched)."""
    from dglke_b200 import _lib
    n0 = eng.h.launch_count()
    if isinstance(batch, dict):
        eng.step_begin(batch["node_ids"], batch["head_local"], batch["tail_local"], batch["rel_ids"], batch["neg_ids"],
                       chunk_size=Cs, neg_sample_size=Ns, neg_head=batch["neg_head"], edge_weight=batch["edge_weight"],
                       next_batch=next_batch)
    else:
        eng.step_begin(batch, chunk_size=Cs, neg_sample_size=Ns, next_batch=next_batch)
    log = eng.step_end()
    _lib.check(eng.lib.kge_rel_apply_dense(eng.h.raw, eng.rel.ref(), rg.data_ptr(), rgs.data_ptr(), float(eng.hp.lr),
                                           eng.h.stream()))
    return log.cpu().numpy(), eng.h.launch_count() - n0


def _batch(n_ent, n_rel, B, Cs, Ns, bounds, seed, neg_head, pool=None, weights=False):
    """Step inputs (CPU int64 tensors) with every id of `bounds` among the heads, the tails and the negatives of the first
    and of the last chunk.  pool: draw entity ids from it (consecutive steps then share rows)."""
    rng = np.random.default_rng(seed)
    C = B // Cs
    draw = (lambda k: rng.choice(pool, k)) if pool is not None else (lambda k: rng.integers(0, n_ent, k))
    h, t, ng = draw(B), draw(B), draw(C * Ns)
    nb = len(bounds)
    h[rng.choice(B, nb, replace=False)] = bounds
    t[rng.choice(B, nb, replace=False)] = bounds
    ng[:nb] = bounds
    ng[-nb:] = bounds[::-1]
    nodes, inv = np.unique(np.concatenate([h, t]), return_inverse=True)
    T = lambda a: th.from_numpy(np.ascontiguousarray(a.astype(np.int64)))
    w = th.from_numpy(rng.uniform(0.5, 1.5, B).astype(np.float32)) if weights else None
    return dict(node_ids=T(nodes), head_local=T(inv[:B]), tail_local=T(inv[B:]), rel_ids=T(rng.integers(0, n_rel, B)),
                neg_ids=T(ng), neg_head=neg_head, edge_weight=w), C


def _on_device(si):
    return {k: (v.cuda() if th.is_tensor(v) else v) for k, v in si.items()}


def _oracle(hp, tables, si, C, Cs, Ns, stale_ent=None, fp64=False):
    """One oracle step from `tables` (not modified).  stale_ent: the entity table the step reads its rows from (rows staged
    one step early); the updates land on `tables` either way."""
    cast = (lambda x: x.double().clone()) if fp64 else (lambda x: x.clone())
    t = [cast(x) for x in tables]
    read = t[0] if stale_ent is None else cast(stale_ent)
    w = si["edge_weight"]
    if w is not None and fp64:
        w = w.double()
    fb = ko.forward_backward(hp, read, t[2], si["node_ids"], si["head_local"], si["tail_local"], si["rel_ids"],
                             si["neg_ids"], C, Cs, Ns, si["neg_head"], w)
    with th.no_grad():
        ko.adagrad_entry(t[0], t[1], si["node_ids"], fb["nodes_grad"], hp.lr)
        ko.adagrad_entry(t[0], t[1], si["neg_ids"], fb["negs_grad"], hp.lr)
        ko.adagrad_entry(t[2], t[3], si["rel_ids"], fb["rels_grad"], hp.lr)
    return dict(pos_score=fb["pos_score"].numpy(), neg_score=fb["neg_score"].numpy(), log=fb["log"],
                nodes_grad=fb["nodes_grad"].numpy(), negs_grad=fb["negs_grad"].numpy(), rels_grad=fb["rels_grad"].numpy(),
                ent_emb=t[0].numpy(), ent_state=t[1].numpy(), rel_emb=t[2].numpy(), rel_state=t[3].numpy())


def _tables(tab, r, rs):
    e, es = tab.read()
    return [e, es, r.cpu(), rs.cpu()]


def _check_tables_and_log(hp, got_log, after, before, si, C, Cs, Ns, stale_ent=None):
    got = dict(log=got_log, e=after[0].numpy(), es=after[1].numpy(), r=after[2].numpy(), rs=after[3].numpy())
    ref = _oracle(hp, before, si, C, Cs, Ns, stale_ent)
    _check_step(hp, got, ref, lambda: _oracle(hp, before, si, C, Cs, Ns, stale_ent, fp64=True), TOL, keys=FUSED_KEYS)


# (model, hidden, gamma, double_ent, double_rel, n_ent, n_rel, B, Cs, Ns, adversarial)
SHAPES = [
    ("TransE_l2", 400, 19.9, False, False, 14951, 1345, 1000, 200, 200, True),   # BASELINE shape
    ("DistMult", 400, 143.0, False, False, 14951, 1345, 1000, 200, 200, True),
    ("ComplEx", 400, 143.0, True, True, 14951, 1345, 1000, 200, 200, True),      # D = 800: per-lane red.add.sys updates
    ("TransE_l2", 512, 19.9, False, False, 4999, 100, 1000, 200, 200, True),     # D = 512: the widest bulk-reduction row
    ("TransE_l2", 516, 19.9, False, False, 4999, 100, 1000, 200, 200, True),     # the first row past it
    ("RotatE", 200, 12.0, True, False, 4999, 53, 1000, 200, 200, True),          # fp32 tiles
    ("TransE_l1", 400, 19.9, False, False, 4999, 100, 400, 200, 200, True),      # fp32 tiles
    ("RESCAL", 64, 12.0, False, False, 2001, 20, 128, 64, 64, False),
]
_sid = lambda c: "%s_d%d%s_B%d_%dx%d" % (c[0], c[1], "_de" if c[3] else "", c[7], c[8], c[9])


def _hyper(cfg, reg_coef=1e-6, lr=0.1):
    model, hidden, gamma, de, dr = cfg[:5]
    return ko.Hyper(model=model, hidden_dim=hidden, gamma=gamma, lr=lr, reg_coef=reg_coef, reg_norm=3, adversarial=cfg[10],
                    adv_temperature=1.0, double_ent=de, double_rel=dr)


def _init(hp, n_ent, n_rel, seed=3):
    ent, es, rel, rs = ko.init_tables(hp, n_ent, n_rel, seed=seed)
    es.uniform_(0.0, 1e-3)          # non-trivial Adagrad state
    rs.uniform_(0.0, 1e-3)
    return ent, es, rel, rs


# ---- A: the 3-call API, stage by stage --------------------------------------------------------------------------------
A_CASES = [(cfg, nh, (2, 3, 8)[(i + nh) % 3]) for i, cfg in enumerate(SHAPES) for nh in (False, True)]


@pytest.mark.parametrize("cfg,neg_head,n_shards", A_CASES,
                         ids=["%s_%s_k%d" % (_sid(c), "head" if nh else "tail", k) for c, nh, k in A_CASES])
def test_forward_backward_and_update_on_sharded_table(cfg, neg_head, n_shards, sharded):
    """Scores, the node / negative / relation gradients (the negatives' through the hi + lo rebuild of their rows in
    k_fused<N>), the log scalars and the updated tables and state."""
    from dglke_b200 import _lib
    hp = _hyper(cfg)
    n_ent, n_rel, B, Cs, Ns = cfg[5:10]
    ent, es, rel, rs = _init(hp, n_ent, n_rel)
    tab = sharded(ent, es, n_shards)
    eng, r, r_s = _engine(hp, tab, rel, rs)
    si, C = _batch(n_ent, n_rel, B, Cs, Ns, tab.boundary_ids(), seed=11, neg_head=neg_head)
    sd = _on_device(si)
    log4 = eng.forward_backward(sd["node_ids"], sd["head_local"], sd["tail_local"], sd["rel_ids"], sd["neg_ids"], Cs, Ns,
                                neg_head)
    U, D = si["node_ids"].numel(), hp.entity_dim
    got = dict(pos=eng.read(_lib.BUF_POS_SCORE, (B,)).cpu().numpy(), neg=eng.read(_lib.BUF_NEG_SCORE, (B, Ns)).cpu().numpy(),
               gn=eng.read(_lib.BUF_NODE_GRAD, (U, D)).cpu().numpy(), gg=eng.read(_lib.BUF_NEG_GRAD, (C * Ns, D)).cpu().numpy(),
               gr=eng.read(_lib.BUF_REL_GRAD, (B, hp.relation_dim)).cpu().numpy(), log=log4.cpu().numpy())
    eng.update()
    e, e_s = tab.read()
    got.update(e=e.numpy(), es=e_s.numpy(), r=r.cpu().numpy(), rs=r_s.cpu().numpy())
    tables = (ent, es, rel, rs)
    ref = _oracle(hp, tables, si, C, Cs, Ns)
    # rows of 800 floats: the wgmma scores of one shard and of several alike are off the float64 oracle by up to
    # 7e-6 of the largest score (test_gpu_parity's 2e-6 floor is set at D <= 400)
    floor = 2e-6 if D <= 512 else 1e-5
    _check_step(hp, got, ref, lambda: _oracle(hp, tables, si, C, Cs, Ns, fp64=True), TOL, score_floor=floor)


# ---- B: the fused step in two halves, deferred relations (ShardedTrainer.step with one rank) ---------------------------
B_CASES = [(cfg, (3, 8, 2)[i % 3], False) for i, cfg in enumerate(SHAPES)]
B_CASES += [(("DistMult", 128, 143.0, False, False, 100003, 1345, 48000, 240, 240, True), 3, False),   # persistent loop
            (SHAPES[0], 8, True)]                                                                          # edge weights


@pytest.mark.parametrize("cfg,n_shards,weighted", B_CASES,
                         ids=["%s_k%d%s" % (_sid(c), k, "_weighted" if w else "") for c, k, w in B_CASES])
def test_fused_step_with_deferred_relations_on_sharded_table(cfg, n_shards, weighted, sharded):
    """Three alternating steps; each is checked against the oracle run from the tables the device had before it.  The
    relation table must move: its gradients reach the caller's buffers for every model."""
    hp = _hyper(cfg)
    n_ent, n_rel, B, Cs, Ns = cfg[5:10]
    ent, es, rel, rs = _init(hp, n_ent, n_rel)
    tab = sharded(ent, es, n_shards)
    eng, r, r_s = _engine(hp, tab, rel, rs)
    rg, rgs = _deferred(eng, n_rel, hp.relation_dim)
    for s in range(3):
        si, C = _batch(n_ent, n_rel, B, Cs, Ns, tab.boundary_ids(), seed=100 + s, neg_head=s % 2 == 1, weights=weighted)
        before = _tables(tab, r, r_s)
        log, _ = _sharded_step(eng, rg, rgs, _on_device(si), Cs, Ns)
        after = _tables(tab, r, r_s)
        moved = float((after[2] - before[2]).abs().max())
        assert moved > 1e-4, "step %d: the relation table did not move (max |delta| %.3e)" % (s, moved)
        _check_tables_and_log(hp, log, after, before, si, C, Cs, Ns)
    assert float(rgs.abs().max()) == 0.0 and float(rg.abs().max()) == 0.0, "relation sums not consumed"


# ---- C: the prefetch pipeline (--async_update) ------------------------------------------------------------------------
def _pool(tab, n_ent, seed, k=500):
    """a few hundred entity ids and the shard boundaries: consecutive batches share most of their rows"""
    return np.union1d(np.random.default_rng(seed).choice(n_ent, k, replace=False), tab.boundary_ids())


def _assert_lag_is_visible(hp, stale_ent, before, si, C, Cs, Ns, what):
    """the oracle step that reads current rows must differ from the one that reads `stale_ent` by more than 10x the
    tolerance (both in float64: the fp32 CPU regulariser has been seen off by a factor, see _check_step)"""
    ref = _oracle(hp, before, si, C, Cs, Ns, stale_ent, fp64=True)
    sync = _oracle(hp, before, si, C, Cs, Ns, fp64=True)
    scale = float(np.abs(ref["ent_emb"]).max())
    diff = float(np.abs(sync["ent_emb"] - ref["ent_emb"]).max())
    assert diff > 10 * (TOL + 5e-6) * scale, "%s: stale and current reads coincide (%.3e), the check is blind" % (what, diff)
    rl, rs = ref["log"]["regularization"], sync["log"]["regularization"]
    assert abs(rs - rl) > 10 * 2e-5 * abs(rl), "%s: the regulariser does not see the stale rows (%g vs %g)" % (what, rl, rs)


PF_SHAPES = [("TransE_l2", 400, 19.9, False, False, 14951, 50, 1000, 200, 200, True),
             ("ComplEx", 400, 143.0, True, True, 14951, 50, 1000, 200, 200, True)]


@pytest.mark.parametrize("cfg", PF_SHAPES, ids=_sid)
def test_prefetch_pipeline_reads_rows_one_step_stale(cfg, sharded):
    """dist_check.py's pipelined mode in one process: steps 1..3 are announced by their predecessor, read the entity rows
    as they were before the previous update (relations current), and launch one kernel fewer (no k_gather_nodes).  The
    regulariser is large enough for the log scalar to show whether the node update used the staged rows."""
    hp = _hyper(cfg, reg_coef=1e-4)
    n_ent, n_rel, B, Cs, Ns = cfg[5:10]
    ent, es, rel, rs = _init(hp, n_ent, n_rel)
    tab = sharded(ent, es, 4)
    eng, r, r_s = _engine(hp, tab, rel, rs)
    rg, rgs = _deferred(eng, n_rel, hp.relation_dim)
    pool = _pool(tab, n_ent, 5)
    steps = 5
    batches = [_batch(n_ent, n_rel, B, Cs, Ns, tab.boundary_ids(), 200 + s, s % 2 == 1, pool=pool)[0] for s in range(steps)]
    dev = [_on_device(si) for si in batches]
    announced = [0 < s < steps - 1 for s in range(steps)]
    snaps, launches = [], []
    for s in range(steps):
        nxt = (dev[s + 1]["node_ids"], dev[s + 1]["neg_ids"]) if s + 1 < steps and announced[s + 1] else None
        before = _tables(tab, r, r_s)
        log, n = _sharded_step(eng, rg, rgs, dev[s], Cs, Ns, next_batch=nxt)
        launches.append(n)
        stale = snaps[s - 1][0] if announced[s] else None
        _check_tables_and_log(hp, log, _tables(tab, r, r_s), before, batches[s], B // Cs, Cs, Ns, stale)
        if announced[s]:
            _assert_lag_is_visible(hp, stale, before, batches[s], B // Cs, Cs, Ns, "step %d" % s)
        snaps.append(before)
    # step 0 also zero-fills the node-gradient region once; the last step gathers its own rows
    assert all(launches[s] == launches[-1] - 1 for s in range(steps) if announced[s]), \
        "staged rows were not used: launches per step %r" % (launches,)


def test_prefetch_of_a_device_sampled_batch(sharded):
    """A DeviceSampler batch announced as such: its node count is known only on the device.  The oracle runs the
    HostSampler's bit-identical batches."""
    from dglke_b200.sampler import DeviceSampler, HostSampler
    cfg = PF_SHAPES[0]
    hp = _hyper(cfg, reg_coef=1e-4)
    n_ent, n_rel, B, Ns = 14951, 50, 1000, 200
    ent, es, rel, rs = _init(hp, n_ent, n_rel)
    tab = sharded(ent, es, 3)
    eng, r, r_s = _engine(hp, tab, rel, rs)
    rg, rgs = _deferred(eng, n_rel, hp.relation_dim)
    rng = np.random.default_rng(9)
    pool = _pool(tab, n_ent, 9, k=300)
    heads, tails, rels = rng.choice(pool, 20000), rng.choice(pool, 20000), rng.integers(0, n_rel, 20000)
    ds = DeviceSampler(heads, rels, tails, n_ent, B, Ns, seed=7)
    hs = HostSampler(heads, rels, tails, n_ent, B, Ns, seed=7)
    Cs, C = ds.chunk_size, ds.num_chunks
    steps, snaps, launches = 4, [], []
    staged = [0 < s < steps - 1 for s in range(steps)]         # the last step gathers: the launch-count reference
    ahead = ds.sample(0)
    for s in range(steps):
        b, ahead = ahead, (ds.sample(s + 1) if s + 1 < steps else None)
        hb = hs.sample(s)
        T = lambda a: th.from_numpy(np.ascontiguousarray(a, dtype=np.int64))
        si = dict(node_ids=T(hb["node_ids"]), head_local=T(hb["head_local"]), tail_local=T(hb["tail_local"]),
                  rel_ids=T(hb["rel"]), neg_ids=T(hb["neg"]), neg_head=hb["neg_head"], edge_weight=None)
        before = _tables(tab, r, r_s)
        log, n = _sharded_step(eng, rg, rgs, b, Cs, Ns, next_batch=ahead if s + 1 < steps and staged[s + 1] else None)
        launches.append(n)
        for got, want in zip(b.tensors(), (si[k] for k in ("node_ids", "head_local", "tail_local", "rel_ids", "neg_ids"))):
            assert th.equal(got.cpu(), want), "device and host sampler disagree at step %d" % s
        assert b.neg_head == si["neg_head"]
        stale = snaps[s - 1][0] if staged[s] else None
        _check_tables_and_log(hp, log, _tables(tab, r, r_s), before, si, C, Cs, Ns, stale)
        if staged[s]:
            _assert_lag_is_visible(hp, stale, before, si, C, Cs, Ns, "step %d" % s)
        snaps.append(before)
    assert launches[1:] == [launches[-1] - 1] * (steps - 2) + [launches[-1]], "launches per step %r" % (launches,)


def test_prefetch_dropped_for_another_batch_and_on_regrowth(sharded):
    """Step 1 runs a batch other than the one step 0 announced: it gathers and reads current rows.  Step 2 announces a
    batch with more negatives (208 per chunk), so the staging buffers regrow and the rows staged for step 2 are dropped:
    step 2 also gathers and reads current rows.  Step 3 reads the rows step 2 staged; step 4 is not announced."""
    cfg = PF_SHAPES[0]
    hp = _hyper(cfg, reg_coef=1e-4)
    n_ent, n_rel, B, Cs = 14951, 50, 1000, 200
    ent, es, rel, rs = _init(hp, n_ent, n_rel)
    tab = sharded(ent, es, 4)
    eng, r, r_s = _engine(hp, tab, rel, rs)
    rg, rgs = _deferred(eng, n_rel, hp.relation_dim)
    pool = _pool(tab, n_ent, 13)
    mk = lambda Ns, seed, nh: _batch(n_ent, n_rel, B, Cs, Ns, tab.boundary_ids(), seed, nh, pool=pool)[0]
    announced_only = _on_device(mk(200, 300, True))            # announced by step 0, never run
    batches = [mk(200, 301, False), mk(200, 302, True), mk(200, 303, False), mk(208, 304, True), mk(208, 305, False)]
    dev = [_on_device(si) for si in batches]
    nxt = [(announced_only["node_ids"], announced_only["neg_ids"]), (dev[2]["node_ids"], dev[2]["neg_ids"]),
           (dev[3]["node_ids"], dev[3]["neg_ids"]), None, None]
    staged = [False, False, False, True, False]
    snaps, launches = [], []
    for s, si in enumerate(batches):
        C = B // Cs
        Ns = si["neg_ids"].numel() // C
        before = _tables(tab, r, r_s)
        log, n = _sharded_step(eng, rg, rgs, dev[s], Cs, Ns, next_batch=nxt[s])
        launches.append(n)
        stale = snaps[s - 1][0] if staged[s] else None
        _check_tables_and_log(hp, log, _tables(tab, r, r_s), before, si, C, Cs, Ns, stale)
        if staged[s]:
            _assert_lag_is_visible(hp, stale, before, si, C, Cs, Ns, "step %d" % s)
        snaps.append(before)
    g = launches[4]                  # step 0 also zero-fills the node-gradient region once
    assert launches[1:] == [g, g, g - 1, g], "launches per step %r" % (launches,)


def test_no_prefetch_when_the_geometry_leaves_no_slots(sharded):
    """d = 1792 with 200-wide chunks: the fused kernels' ring leaves fewer than 2 row slots per prefetch warp, so an
    announced batch is not staged and every step gathers current rows."""
    cfg = ("DistMult", 1792, 143.0, False, False, 4001, 20, 1000, 200, 200, True)
    hp = _hyper(cfg, reg_coef=1e-4)
    n_ent, n_rel, B, Cs, Ns = cfg[5:10]
    ent, es, rel, rs = _init(hp, n_ent, n_rel)
    tab = sharded(ent, es, 4)
    eng, r, r_s = _engine(hp, tab, rel, rs)
    rg, rgs = _deferred(eng, n_rel, hp.relation_dim)
    pool = _pool(tab, n_ent, 17)
    batches = [_batch(n_ent, n_rel, B, Cs, Ns, tab.boundary_ids(), 400 + s, s % 2 == 1, pool=pool)[0] for s in range(4)]
    dev = [_on_device(si) for si in batches]
    launches = []
    for s in range(4):
        nxt = (dev[s + 1]["node_ids"], dev[s + 1]["neg_ids"]) if s + 1 < 3 else None
        before = _tables(tab, r, r_s)
        log, n = _sharded_step(eng, rg, rgs, dev[s], Cs, Ns, next_batch=nxt)
        launches.append(n)
        _check_tables_and_log(hp, log, _tables(tab, r, r_s), before, batches[s], B // Cs, Cs, Ns)
    # step 0 zero-fills the node-gradient region once; step 3 was not announced
    assert launches[1:] == [launches[3]] * 3, "launches per step %r" % (launches,)


# ---- D: stand-alone ops -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_shards,D", [(3, 400), (8, 516)])
def test_gather_and_adagrad_on_sharded_table(n_shards, D, sharded):
    """kge_gather bit exact; kge_adagrad with duplicated ids (system-scope atomics on state and rows) against the oracle."""
    import ctypes as C
    from dglke_b200 import _lib
    n = 14951
    g = th.Generator().manual_seed(n_shards)
    emb, state = th.randn(n, D, generator=g) * 0.1, th.rand(n, generator=g) * 1e-3
    tab = sharded(emb, state, n_shards)
    rng = np.random.default_rng(D)
    bounds = tab.boundary_ids()
    idx = np.concatenate([rng.integers(0, n, 3000), bounds, bounds, rng.integers(0, 40, 200)])   # duplicates
    rng.shuffle(idx)
    idx_c = th.from_numpy(idx)
    idx_d = idx_c.cuda()
    h = _handle()
    out = th.empty((len(idx), D), dtype=th.float32, device=idx_d.device)
    _lib.check(h.lib.kge_gather(h.raw, tab.table.ref(), idx_d.data_ptr(), len(idx), out.data_ptr(), h.stream()))
    assert th.equal(out.cpu(), emb[idx_c])
    grad = th.randn(len(idx), D, generator=g)
    e2, s2 = emb.clone(), state.clone()
    ko.adagrad_entry(e2, s2, idx_c, grad, 0.3)
    gd = grad.cuda()
    _lib.check(h.lib.kge_adagrad(h.raw, tab.table.ref(), idx_d.data_ptr(), gd.data_ptr(), len(idx), C.c_float(0.3),
                                 h.stream()))
    e, s = tab.read()
    np.testing.assert_allclose(e.numpy(), e2.numpy(), rtol=2e-5, atol=1e-7)
    np.testing.assert_allclose(s.numpy(), s2.numpy(), rtol=2e-5, atol=1e-9)


def test_nine_shards_are_refused():
    from dglke_b200 import _lib
    from dglke_b200.engine import DeviceTable
    shards = [th.zeros(2, 4, device="cuda") for _ in range(9)]
    states = [th.zeros(2, device="cuda") for _ in range(9)]
    tab = DeviceTable(shards, states, 18, 4, devices=[0] * 9)
    h = _handle()
    idx = th.arange(18, device="cuda")
    out = th.empty(18, 4, device="cuda")
    with pytest.raises(_lib.KgeError, match="n_shards=9"):
        _lib.check(h.lib.kge_gather(h.raw, tab.ref(), idx.data_ptr(), 18, out.data_ptr(), h.stream()))
