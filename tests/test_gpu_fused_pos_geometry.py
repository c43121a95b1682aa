"""k_fused<P> at every (GEMM1 width NV, GEMM2 chunk width NW) pair that geometry() picks, with and without prefetch slots.

NV is the wgmma N of GEMM1 (64 / 128 / 208 / 256 from the chunk's negatives Ns).  NW is the output-column chunk of
GEMM2 (GA = V.Bn): 200 where ceil(D / 200) * 200 < ceil(D / 128) * 128, else 128, and always 128 at NV = 256, where
the V buffer (128 KB) and two 200-column stages would not fit the ring.  The D values below put both widths at one,
two, three and four chunks, with a last chunk that is full, nearly full or nearly empty; each Ns value is one NV.  The
fused path stops at Ns = 240 (fused_supported), so NV = 256 is taken with Ns = 240.

One TransE_l2 step (its column sums of V go through the hand-off warps as well) against the oracle at the hot-shape
tolerances of DESIGN.md §2: scores, log scalars, node gradients (which carry GA), negative gradients (which carry the
V^T slabs), relation gradients, and the tables and Adagrad state after the update.  k_fused<P>'s launch name reports
the variant and the ring layout that ran (NV, NW, prefetch slots per warp, V hand-off warps); each case asserts it
against the rule below, so a geometry() that picked another width would fail here rather than test something else.

With prefetch slots (sharded tables, the next batch announced) the ring stays at 192 KB: NW = 200 still fits next to the
V buffer at NV = 64 and 128, not at 208.  Those layouts run the pipelined sharded step of test_gpu_sharded.py, whose
rows are one step stale, at d = 400."""
import pytest

import kge_oracle as ko
from test_gpu_parity import _random_step, _run_and_check
from test_gpu_sharded import (sharded, _hyper, _init, _engine, _deferred, _pool, _batch, _on_device,   # noqa: F401
                              _sharded_step, _tables, _check_tables_and_log)

DS = [32, 40, 128, 200, 392, 400, 408, 800]
NSS = [64, 128, 200, 240]
CS = 200           # two row tiles per chunk, the second one ragged (72 rows)


def _widths(D, Ns):
    nv = 64 if Ns <= 64 else (128 if Ns <= 128 else (208 if Ns <= 208 else 256))
    nw = 200 if nv < 256 and (D + 199) // 200 * 200 < (D + 127) // 128 * 128 else 128
    return nv, nw


def test_width_rule_covers_every_pair():
    """The grid reaches every (NV, NW) pair the kernel is instantiated for, and both widths at more than one chunk."""
    pairs = {_widths(D, Ns) for D in DS for Ns in NSS}
    assert pairs == {(64, 128), (64, 200), (128, 128), (128, 200), (208, 128), (208, 200), (256, 128)}, pairs
    assert {(D + nw - 1) // nw for D in DS for nw in (128, 200) if _widths(D, 64)[1] == nw} >= {1, 2, 4}


@pytest.mark.gpu
@pytest.mark.parametrize("Ns", NSS)
@pytest.mark.parametrize("D", DS)
def test_fused_step_at_every_chunk_geometry(D, Ns):
    from dglke_b200 import _lib
    nv, nw = _widths(D, Ns)
    hp = ko.Hyper(model="TransE_l2", hidden_dim=D, gamma=19.9, lr=0.1, reg_coef=1e-6, reg_norm=3, adversarial=True,
                  adv_temperature=1.0)
    n_ent, n_rel, B = 6000, 50, 2 * CS
    ent, es, rel, rs = ko.init_tables(hp, n_ent, n_rel, seed=5)
    es.uniform_(0.0, 1e-3)
    rs.uniform_(0.0, 1e-3)
    si, C = _random_step(hp, n_ent, n_rel, B, CS, Ns, neg_head=bool(D % 2 == 0 and Ns % 3 == 0), seed=D * 1000 + Ns)
    o_ent, o_es, o_rel, o_rs = ent.clone(), es.clone(), rel.clone(), rs.clone()
    fb = ko.train_step(hp, o_ent, o_es, o_rel, o_rs, si["node_ids"], si["head_local"], si["tail_local"],
                       si["rel_ids"], si["neg_ids"], C, CS, Ns, si["neg_head"])
    ref = dict(pos_score=fb["pos_score"].numpy(), neg_score=fb["neg_score"].numpy(), log=fb["log"],
               nodes_grad=fb["nodes_grad"].numpy(), negs_grad=fb["negs_grad"].numpy(),
               rels_grad=fb["rels_grad"].numpy(), ent_emb=o_ent.numpy(), ent_state=o_es.numpy(),
               rel_emb=o_rel.numpy(), rel_state=o_rs.numpy())
    h = _lib.get_handle(0)
    h.profile_enable(True)
    try:
        _run_and_check(hp, (ent, es, rel, rs), si, C, CS, Ns, ref, tol=5e-5)
        names = [n for n, _ in h.profile_read()]
    finally:
        h.profile_enable(False)
    pos = [n for n in names if n.startswith("k_fused<P")]
    assert pos and all(n.endswith(" NV=%d NW=%d pf=0 hand=3" % (nv, nw)) for n in pos), (nv, nw, names)
    assert any(n.startswith("k_fused<N") for n in names), names


# (Ns, NV, NW, prefetch slots per warp) at d = 400 with prefetch: the ring keeps 192 KB; 1 hand-off warp
PF_CASES = [(64, 64, 200, 8), (128, 128, 200, 8), (200, 208, 128, 7)]


@pytest.mark.gpu
@pytest.mark.parametrize("Ns,nv,nw,slots", PF_CASES, ids=["Ns%d_NV%d_NW%d" % c[:3] for c in PF_CASES])
def test_prefetch_layouts(Ns, nv, nw, slots, sharded):
    """Pipelined sharded step (4 shards, deferred relations): steps 1 and 2 are announced by their predecessor and read
    the rows it staged, one step stale.  Every step against the oracle; the announcing steps run k_fused<P> with the
    prefetch layout, the others with the 223 KB ring."""
    cfg = ("TransE_l2", 400, 19.9, False, False, 14951, 50, 1000, CS, Ns, True)
    hp = _hyper(cfg, reg_coef=1e-4)
    n_ent, n_rel, B, Cs = cfg[5:9]
    ent, es, rel, rs = _init(hp, n_ent, n_rel)
    tab = sharded(ent, es, 4)
    eng, r, r_s = _engine(hp, tab, rel, rs)
    rg, rgs = _deferred(eng, n_rel, hp.relation_dim)
    pool = _pool(tab, n_ent, 7)
    steps = 4
    batches = [_batch(n_ent, n_rel, B, Cs, Ns, tab.boundary_ids(), 300 + s, s % 2 == 1, pool=pool)[0] for s in range(steps)]
    dev = [_on_device(si) for si in batches]
    announced = [0 < s < steps - 1 for s in range(steps)]
    snaps = []
    eng.h.profile_enable(True)
    try:
        for s in range(steps):
            nxt = (dev[s + 1]["node_ids"], dev[s + 1]["neg_ids"]) if s + 1 < steps and announced[s + 1] else None
            before = _tables(tab, r, r_s)
            eng.h.profile_read()
            log, _ = _sharded_step(eng, rg, rgs, dev[s], Cs, Ns, next_batch=nxt)
            pos = [n for n, _ in eng.h.profile_read() if n.startswith("k_fused<P")]
            want = (" NV=%d NW=%d pf=%d hand=1" % (nv, nw, slots)) if nxt is not None else \
                   (" NV=%d NW=%d pf=0 hand=3" % _widths(400, Ns))
            assert pos and all(n.endswith(want) for n in pos), (s, want, pos)
            stale = snaps[s - 1][0] if announced[s] else None
            _check_tables_and_log(hp, log, _tables(tab, r, r_s), before, batches[s], B // Cs, Cs, Ns, stale)
            snaps.append(before)
    finally:
        eng.h.profile_enable(False)
