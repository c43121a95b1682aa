"""The fused step's register-side GEMM operands: A (GEMM1 of k_fused<P>) and V^T (the GEMM of k_fused<N>) are stored once
as fp32 and split into TF32 hi/lo by the MMA warps, per k-step, from shared memory.

- One kge_step_fused at a ragged shape (Cs = 200, so the second 128-row tile of positives holds 72 rows, and D = 408, so
  the last 32-column k-block of GEMM1 runs 3 of its 4 k-steps) against float64, through the step-increment harness of
  tests/test_gpu_step_increments.py (same bounds); the benchmark's own shape is one of that file's cases.
- Every (NV, NW) pair of k_fused<P> and every output-column width of k_fused<N> runs once (launch names), one TransE_l2
  step each against the oracle.  The 256-wide variants read their A operand as hi/lo slabs from shared memory.
- The compiler's log of kge_fused.cu (written by the build): all 15 variants build without spills and without
  serialised wgmma."""
import os
import re

import pytest

import kge_oracle as ko
from test_gpu_parity import _random_step, _run_and_check
from test_gpu_step_increments import Case, run_fused_case

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LOG = os.path.join(ROOT, "dgl-ke_b200", "build", "kge_fused.ptxas.log")

RAGGED = Case("TransE_l2_d408_ragged", "TransE_l2", 408, 19.9, 14951, 1345, 1000, 200, 200, reg_coef=4.5e-3)


@pytest.mark.gpu
@pytest.mark.parametrize("neg_head", [False, True])
def test_fused_step_increments_at_a_ragged_shape(neg_head):
    run_fused_case(RAGGED, neg_head)


# (D, Ns) -> k_fused<P> (NV, NW) and k_fused<N> NW, one TransE_l2 step on one GPU with Cs = 200
VARIANTS = [(64, 64, (64, 128), 64), (200, 64, (64, 200), 200), (128, 128, (128, 128), 128), (200, 128, (128, 200), 200),
            (256, 200, (208, 128), 256), (400, 200, (208, 200), 200), (128, 240, (256, 128), 128)]


@pytest.mark.gpu
@pytest.mark.parametrize("D,Ns,pos,neg", VARIANTS, ids=["D%d_Ns%d" % v[:2] for v in VARIANTS])
def test_every_variant_launches(D, Ns, pos, neg):
    from dglke_b200 import _lib
    Cs = 200
    hp = ko.Hyper(model="TransE_l2", hidden_dim=D, gamma=19.9, lr=0.1, reg_coef=1e-6, reg_norm=3, adversarial=True,
                  adv_temperature=1.0)
    n_ent, n_rel, B = 6000, 50, 2 * Cs
    ent, es, rel, rs = ko.init_tables(hp, n_ent, n_rel, seed=11)
    es.uniform_(0.0, 1e-3)
    rs.uniform_(0.0, 1e-3)
    si, C = _random_step(hp, n_ent, n_rel, B, Cs, Ns, neg_head=False, seed=D * 1000 + Ns)
    o_ent, o_es, o_rel, o_rs = ent.clone(), es.clone(), rel.clone(), rs.clone()
    fb = ko.train_step(hp, o_ent, o_es, o_rel, o_rs, si["node_ids"], si["head_local"], si["tail_local"],
                       si["rel_ids"], si["neg_ids"], C, Cs, Ns, si["neg_head"])
    ref = dict(pos_score=fb["pos_score"].numpy(), neg_score=fb["neg_score"].numpy(), log=fb["log"],
               nodes_grad=fb["nodes_grad"].numpy(), negs_grad=fb["negs_grad"].numpy(),
               rels_grad=fb["rels_grad"].numpy(), ent_emb=o_ent.numpy(), ent_state=o_es.numpy(),
               rel_emb=o_rel.numpy(), rel_state=o_rs.numpy())
    h = _lib.get_handle(0)
    h.profile_enable(True)
    try:
        _run_and_check(hp, (ent, es, rel, rs), si, C, Cs, Ns, ref, tol=5e-5)
        names = [n for n, _ in h.profile_read()]
    finally:
        h.profile_enable(False)
    p = [n for n in names if n.startswith("k_fused<P")]
    n = [n for n in names if n.startswith("k_fused<N")]
    assert p and all(x.endswith(" NV=%d NW=%d pf=0 hand=3" % pos) for x in p), (pos, names)
    assert n and all(x.endswith(" NW=%d" % neg) for x in n), (neg, names)


# (kernel, template arguments) of every variant: all must build clean
CLEAN = [("k_fused_pos", "ILi%dELi%dE" % pw) for pw in ((64, 128), (64, 200), (128, 128), (128, 200), (208, 128),
                                                        (208, 200), (256, 128))] + \
        [("k_fused_neg", "ILi%dELb%dE" % (w, f)) for w in (64, 128, 200, 256) for f in (0, 1)]


@pytest.mark.skipif(not os.path.exists(LOG), reason="no compiler log: the library was not built here")
def test_compiler_gate():
    log = open(LOG).read()
    blocks = re.split(r"ptxas info\s+: Compiling entry function ", log)
    seen = set()
    for kern, targs in CLEAN:
        mangled = "%d%s%s" % (len(kern), kern, targs)
        hit = [b for b in blocks if b.startswith("'") and mangled in b.split("'")[1]]
        assert hit, "no compiler output for %s<%s>" % (kern, targs)
        props = hit[0]
        assert "0 bytes spill stores, 0 bytes spill loads" in props.split("Used")[0], (kern, targs, props[:400])
        seen.add(mangled)
    assert len(seen) == 15
    for m in re.finditer(r"\((C75(?:11|12|19|20))\).*?function '([^']+)'", log):
        assert not any(s in m.group(2) for s in seen), "%s for %s" % (m.group(1), m.group(2))
