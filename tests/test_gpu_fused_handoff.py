"""The hand-off of the backward coefficients from k_fused<P> to k_fused<N>.

k_fused<P> writes V_ij as TF32 hi/lo pairs in the transposed slab layout V^T[c][i / 32][j][i % 32], and (TransE_l2) the
column sums sum_i V_ij of each 128-row tile of positives; k_fused<N> computes G_neg = V^T.A from them.  Checked here:
- the coefficients k_fused<N> reads are those k_fused<P> produced, bit for bit (hi + lo of the P-side value);
- the negatives' gradient (KGE_BUF_NEG_GRAD) and the tables after the update against the float64 oracle, at shapes whose
  last 32-row block of positives is partial by 8, 16 or 24 rows, Cs a multiple of 32, Cs != Ns, a single 128-row tile,
  two tiles of positives (two column-sum partials), edge weights, the uniform weighting, DistMult and ComplEx with rows
  of 800 floats;
- three fused steps on a 2-shard table with the prefetch pipeline (the prefetch slots share the ring with the stages).

mean(G_neg^2), which k_fused<N> computes in its epilogue, reaches only the Adagrad state, and from the U(0, 1e-3) state
used here its share of the state is below the tolerance; tests/test_gpu_step_increments.py checks it from a seeded
state."""
import numpy as np
import pytest
import torch as th

import kge_oracle as ko
from test_gpu_parity import _random_step, _engine, _oracle_fp64, _check_step
from test_gpu_sharded import (sharded, _engine as _sharded_engine, _deferred, _sharded_step, _batch, _on_device,  # noqa: F401
                              _tables, _check_tables_and_log, _pool)

pytestmark = pytest.mark.gpu

TOL = 5e-5


def _rna_tf32(x):
    """cvt.rna.tf32.f32: round to 10 mantissa bits, ties away from zero (low 13 bits cleared)"""
    b = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32).astype(np.uint64)
    return ((b + 0x1000) & 0xFFFFE000).astype(np.uint32).view(np.float32)


def _hi_plus_lo(x):
    """the fp32 value the N side rebuilds from the hi/lo pair the P side stores (split_tf32, then hi + lo)"""
    x = np.ascontiguousarray(x, dtype=np.float32)
    hi = _rna_tf32(x)
    lo = _rna_tf32(x - hi)
    return hi + lo


# (model, hidden, double_ent, gamma, B, Cs, Ns, adversarial, weighted)
CASES = [
    ("TransE_l2", 400, False, 19.9, 13200, 200, 200, True, False),   # the benchmark's shape; last i-block 8 rows
    ("TransE_l2", 400, False, 19.9, 1040, 208, 200, True, False),    # last i-block 16 rows
    ("TransE_l2", 96, False, 10.0, 1080, 216, 120, True, False),     # last i-block 24 rows, one 128-row tile of negatives
    ("TransE_l2", 128, False, 10.0, 928, 232, 232, True, False),     # 8 rows, wgmma width 256 on the P side
    ("TransE_l2", 64, False, 10.0, 960, 240, 64, True, False),       # Cs != Ns: 16 rows, one tile of negatives
    ("TransE_l2", 64, False, 10.0, 640, 64, 240, True, False),       # Cs != Ns: one tile of positives, two of negatives
    ("TransE_l2", 400, False, 19.9, 896, 224, 128, True, False),     # Cs a multiple of 32, one tile of negatives
    ("TransE_l2", 400, False, 19.9, 1000, 200, 200, False, False),   # uniform weighting 1 / Ns
    ("TransE_l2", 400, False, 19.9, 1000, 200, 200, True, True),     # edge weights
    ("DistMult", 800, False, 143.0, 600, 200, 200, True, False),
    ("ComplEx", 400, True, 143.0, 600, 200, 200, True, False),       # D = 800
    ("DistMult", 40, False, 5.0, 96, 48, 24, True, False),           # D narrower than one output chunk
]
_cid = lambda c: "%s_d%d%s_B%d_%dx%d%s%s" % (c[0], c[1], "_de" if c[2] else "", c[4], c[5], c[6],
                                            "" if c[7] else "_uniform", "_weighted" if c[8] else "")


@pytest.mark.parametrize("cfg", CASES, ids=_cid)
@pytest.mark.parametrize("neg_head", [False, True])
def test_negative_side_consumes_the_positive_side_coefficients(cfg, neg_head):
    from dglke_b200 import _lib
    model, hidden, de, gamma, B, Cs, Ns, adv, weighted = cfg
    hp = ko.Hyper(model=model, hidden_dim=hidden, gamma=gamma, lr=0.1, reg_coef=1e-6, reg_norm=3, adversarial=adv,
                  adv_temperature=1.0, double_ent=de, double_rel=de)
    n_ent, n_rel = 5003, 101
    ent, es, rel, rs = ko.init_tables(hp, n_ent, n_rel, seed=7)
    es.uniform_(0.0, 1e-3)
    rs.uniform_(0.0, 1e-3)
    si, C = _random_step(hp, n_ent, n_rel, B, Cs, Ns, neg_head, seed=41)
    if weighted:
        si["edge_weight"] = th.from_numpy(np.random.default_rng(42).uniform(0.5, 1.5, B).astype(np.float32))
    tables0 = [x.clone() for x in (ent, es, rel, rs)]
    eng, (e, e_s, r, r_s) = _engine(hp, ent, es, rel, rs)
    dev = eng.device
    dump = th.full((2 * B * Ns,), float("nan"), dtype=th.float32, device=dev)
    eng.h.set_dump(dump)
    try:
        d = lambda t: t.to(dev)
        w = d(si["edge_weight"]) if weighted else None
        log4 = eng.forward_backward(d(si["node_ids"]), d(si["head_local"]), d(si["tail_local"]), d(si["rel_ids"]),
                                    d(si["neg_ids"]), Cs, Ns, neg_head, w)
        gg = eng.read(_lib.BUF_NEG_GRAD, (C * Ns, hp.entity_dim)).cpu().numpy()
        th.cuda.synchronize()
        VP = dump[:B * Ns].cpu().numpy().reshape(B, Ns)
        VN = dump[B * Ns:].cpu().numpy().reshape(C, Ns, Cs).transpose(0, 2, 1).reshape(B, Ns)
    finally:
        eng.h.set_dump(None)
    eng.update()
    th.cuda.synchronize()

    assert not np.isnan(VP).any() and not np.isnan(VN).any(), "coefficients missing from a dump"
    want = _hi_plus_lo(VP)
    diff = VN.view(np.uint32) != want.view(np.uint32)
    assert not diff.any(), "k_fused<N> read %d coefficients other than k_fused<P> wrote, first (row, col): %s" % (
        int(diff.sum()), np.argwhere(diff)[:8].tolist())

    got = dict(gg=gg, log=log4.cpu().numpy(), e=e.cpu().numpy(), es=e_s.cpu().numpy())
    ref64 = _oracle_fp64(hp, tables0, si, C, Cs, Ns)
    _check_step(hp, got, ref64, lambda: ref64, TOL, allow_fp64_arbitration=False, keys=("log", "gg", "e", "es"))


# (model, hidden, double_ent, double_rel, gamma, n_ent, n_rel, B, Cs, Ns, adversarial) as in test_gpu_sharded
PF_CASES = [("TransE_l2", 400, False, False, 19.9, 14951, 50, 1000, 200, 200, True),    # 2 stages of 200 columns
            ("DistMult", 128, False, False, 143.0, 14951, 50, 1000, 200, 200, True),    # 128-column stages, 3 -> 2
            ("TransE_l2", 512, False, False, 19.9, 4999, 50, 1000, 200, 200, True)]     # 200-column chunks, not 256


@pytest.mark.parametrize("cfg", PF_CASES, ids=lambda c: "%s_d%d" % (c[0], c[1]))
def test_three_prefetched_fused_steps_on_two_shards(cfg, sharded):
    """Steps 1 and 2 are announced by their predecessor: both fused kernels copy the next step's rows through the slots
    behind their stages while they compute.  Every step against the oracle from the tables the device had before it."""
    hp = ko.Hyper(model=cfg[0], hidden_dim=cfg[1], gamma=cfg[4], lr=0.1, reg_coef=1e-4, reg_norm=3, adversarial=cfg[10],
                  adv_temperature=1.0, double_ent=cfg[2], double_rel=cfg[3])
    n_ent, n_rel, B, Cs, Ns = cfg[5:10]
    ent, es, rel, rs = ko.init_tables(hp, n_ent, n_rel, seed=3)
    es.uniform_(0.0, 1e-3)
    rs.uniform_(0.0, 1e-3)
    tab = sharded(ent, es, 2)
    eng, r, r_s = _sharded_engine(hp, tab, rel, rs)
    rg, rgs = _deferred(eng, n_rel, hp.relation_dim)
    pool = _pool(tab, n_ent, 5)
    steps = 3
    batches = [_batch(n_ent, n_rel, B, Cs, Ns, tab.boundary_ids(), 300 + s, s % 2 == 1, pool=pool)[0] for s in range(steps)]
    dev = [_on_device(si) for si in batches]
    snaps, launches = [], []
    for s in range(steps):
        nxt = (dev[s + 1]["node_ids"], dev[s + 1]["neg_ids"]) if s + 1 < steps else None
        before = _tables(tab, r, r_s)
        log, n = _sharded_step(eng, rg, rgs, dev[s], Cs, Ns, next_batch=nxt)
        launches.append(n)
        stale = snaps[s - 1][0] if s > 0 else None
        _check_tables_and_log(hp, log, _tables(tab, r, r_s), before, batches[s], B // Cs, Cs, Ns, stale)
        snaps.append(before)
    # step 0 gathers its own rows (and zero-fills the node gradients once); steps 1 and 2 read the staged ones
    assert launches[1] == launches[2] < launches[0], "staged rows were not used: launches per step %r" % (launches,)
