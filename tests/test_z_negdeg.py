"""--neg_deg_sample (SURVEY 8 a6).  CPU: the oracle's restatement is pinned to the reference's fixtures by
tests/test_oracle_golden.py (negdeg_* cases).  GPU: tests/negdeg_check.py, run once in a process of its own."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def negdeg_check():
    return subprocess.run([sys.executable, os.path.join(ROOT, "tests", "negdeg_check.py")], capture_output=True, text=True,
                          timeout=900, cwd=ROOT)


@pytest.mark.gpu
def test_neg_deg_sample_matches_reference_fixtures_and_oracle(negdeg_check):
    out = negdeg_check
    assert "NEGDEG_CHECK_OK" in out.stdout, out.stdout[-3000:] + out.stderr[-3000:]


@pytest.mark.gpu
@pytest.mark.xfail(strict=False, reason="rows with an Adagrad state near 1e-7 amplify fp32 rounding of the gradient past atol 5e-5 "
                                        "(RotatE, 1-3 of 1.2 M elements; the fp32 CPU oracle is as far from float64 as the device)")
def test_neg_deg_sample_fused_step_entity_table(negdeg_check):
    assert "NEGDEG_TABLE_MISS" not in negdeg_check.stdout, negdeg_check.stdout[-3000:]


def test_neg_deg_sample_step_configuration():
    """host side: the flag travels in the step configuration; chunk bookkeeping of the extra columns"""
    from dglke_b200 import _lib
    from dglke_b200.engine import Hyper
    import ctypes as C
    cfg = _lib.make_cfg("TransE_l2", 8, 8, 12.0, 0.1, 0.1, 0.0, 3, False, 1.0, False, 16, 8, 4, neg_deg_sample=True)
    assert cfg.neg_deg_sample == 1 and cfg.neg_sample_size == 4 and C.sizeof(_lib.StepCfg) == 80
    assert _lib.StepCfg.neg_deg_sample.offset == 76
    assert Hyper(neg_deg_sample=True).neg_deg_sample and not Hyper().neg_deg_sample


@pytest.mark.parametrize("model,de", [("TransE_l2", False), ("DistMult", False), ("RotatE", True), ("RESCAL", False)])
@pytest.mark.parametrize("neg_head", [False, True])
def test_fixup_algebra_of_kge_negdeg_equals_the_reference_semantics(model, de, neg_head):
    """CPU emulation of what kge_negdeg.cu does around the UNCHANGED step, against the oracle's restatement of the
    reference (which tests/test_oracle_golden.py pins to the reference's fixtures):

      ordinary step over the augmented id list ids' (own rows | sampled rows, all treated as one traced negative tensor
      with its regulariser terms) + masked diagonal  -->  fix-ups: drop the prepended rows' regulariser log share, move
      (their gradient - reg'(row)) onto the positive node they are a copy of, zero their gradient rows (the negative Adagrad
      entry then adds 0 to their state and rows)."""
    import numpy as np
    import torch as th
    import kge_oracle as ko
    hp = ko.Hyper(model=model, hidden_dim=8, gamma=6.0, lr=0.2, reg_coef=1e-3, reg_norm=3, adversarial=True,
                  adv_temperature=0.7, double_ent=de, neg_deg_sample=True)
    plain = ko.Hyper(**{**hp.__dict__, "neg_deg_sample": False})
    n_ent, n_rel, B, Cs, Ns = 25, 3, 12, 4, 6
    C, Nse = B // Cs, Cs + Ns
    ent0, es0, rel0, rs0 = ko.init_tables(hp, n_ent, n_rel, seed=2)
    es0 += 0.05
    rng = np.random.default_rng(7)
    h, t = rng.integers(0, n_ent, B), rng.integers(0, n_ent, B)
    nodes, inv = np.unique(np.concatenate([h, t]), return_inverse=True)
    T = lambda a: th.from_numpy(np.ascontiguousarray(np.asarray(a, dtype=np.int64)))
    node_ids, hl, tl, rel_ids, neg_ids = T(nodes), T(inv[:B]), T(inv[B:]), T(rng.integers(0, n_rel, B)), T(rng.integers(0, n_ent, C * Ns))

    # ---- the reference semantics
    want = [x.clone() for x in (ent0, es0, rel0, rs0)]
    fb = ko.train_step(hp, *want, node_ids, hl, tl, rel_ids, neg_ids, C, Cs, Ns, neg_head)

    # ---- the emulated device flow
    own = node_ids[hl if neg_head else tl].reshape(C, Cs)                        # k_negdeg_ids
    ids2 = th.cat([own, neg_ids.reshape(C, Ns)], 1).reshape(-1)
    nodes_l = ent0[node_ids].clone().requires_grad_(True)
    rels_l = rel0[rel_ids].clone().requires_grad_(True)
    negs_l = ent0[ids2].clone().requires_grad_(True)                             # ONE traced tensor of C * (Cs + Ns) rows
    hh, tt = nodes_l[hl], nodes_l[tl]
    pos = ko.positive_score(plain, hh, rels_l, tt)
    neg = (ko.negative_score(plain, negs_l, rels_l, tt, C, Cs, Nse, True) if neg_head
           else ko.negative_score(plain, hh, rels_l, negs_l, C, Cs, Nse, False))
    mask = th.ones(C, Cs, Nse)
    mask[:, th.arange(Cs), th.arange(Cs)] = 0                                    # k_negdeg_mask_scores / _mask_coef
    loss, log = ko.loss_terms(plain, pos, (neg * mask).reshape(B, Nse))
    reg_rows = th.cat([nodes_l, negs_l], 0)
    reg = hp.reg_coef * (reg_rows.abs().pow(3).sum() + rels_l.abs().pow(3).sum())
    (loss + reg).backward()
    is_own = th.zeros(C, Nse, dtype=th.bool)
    is_own[:, :Cs] = True
    is_own = is_own.reshape(-1)
    reg_log = float(reg.detach()) - hp.reg_coef * float(negs_l.detach()[is_own].abs().pow(3).sum())     # k_negdeg_zero_reg
    g_nodes, g_negs = nodes_l.grad.clone(), negs_l.grad.clone()
    x_own = negs_l.detach()[is_own]
    moved = g_negs[is_own] - 3.0 * hp.reg_coef * x_own.abs() * x_own                                      # k_negdeg_scatter
    g_nodes.index_add_(0, (hl if neg_head else tl), moved)
    g_negs[is_own] = 0
    got = [x.clone() for x in (ent0, es0, rel0, rs0)]
    ko.adagrad_entry(got[0], got[1], node_ids, g_nodes, hp.lr)
    ko.adagrad_entry(got[0], got[1], ids2, g_negs, hp.lr)            # prepended rows: state += 0, row += 0
    ko.adagrad_entry(got[2], got[3], rel_ids, rels_l.grad, hp.lr)

    np.testing.assert_allclose(float(loss.detach()), fb["log"]["loss"], rtol=1e-6)
    np.testing.assert_allclose(reg_log, fb["log"]["regularization"], rtol=1e-5)
    np.testing.assert_allclose(g_nodes.numpy(), fb["nodes_grad"].numpy(), rtol=1e-4, atol=1e-7)
    np.testing.assert_allclose(g_negs.reshape(C, Nse, -1)[:, Cs:].reshape(C * Ns, -1).numpy(), fb["negs_grad"].numpy(), rtol=1e-5, atol=1e-8)
    for a, b in zip(got, want):
        np.testing.assert_allclose(a.numpy(), b.numpy(), rtol=1e-5, atol=1e-7)


def test_predict_neg_score_and_forward_test_logic_with_a_cpu_stand_in():
    """KEModel.predict_neg_score / forward_test are thin glue over the score kernels: run the glue itself on the CPU with
    the oracle's score functions standing in for the kernels -- default path (must be the plain chunked score) and the
    neg_deg_sample path (reference semantics: own rows first, masked diagonal, neg_sample_size updated)."""
    import types
    import numpy as np
    import torch as th
    import kge_oracle as ko
    from dglke_b200.general_models import KEModel
    from dglke_b200.graph import build_pos_graph, NegGraph
    hp = ko.Hyper(model="DistMult", hidden_dim=8, gamma=12.0)
    ent, _, rel, _ = ko.init_tables(hp, 40, 3, seed=1)
    fake = types.SimpleNamespace(
        entity_emb=lambda ids, gpu_id, trace: ent[ids], relation_emb=lambda ids, gpu_id, trace: rel[ids],
        head_neg_prepare=lambda rid, C, a, b, gpu_id, trace: (a, b), tail_neg_prepare=lambda rid, C, a, b, gpu_id, trace: (a, b),
        head_neg_score=lambda hn, r, t, C, Cs, Ns: ko.negative_score(hp, hn, r, t, C, Cs, Ns, True),
        tail_neg_score=lambda h, r, tn, C, Cs, Ns: ko.negative_score(hp, h, r, tn, C, Cs, Ns, False),
        args=types.SimpleNamespace(eval_filter=False, neg_deg_sample_eval=False))
    fake.predict_score = lambda g: ko.positive_score(hp, g.ndata["emb"][g.all_edges()[0]], g.edata["emb"], g.ndata["emb"][g.all_edges()[1]])
    fake.predict_neg_score = lambda *a, **k: KEModel.predict_neg_score(fake, *a, **k)
    rng = np.random.default_rng(0)
    C, Cs, Ns = 2, 4, 6
    H, R, T_ = rng.integers(0, 40, C * Cs), rng.integers(0, 3, C * Cs), rng.integers(0, 40, C * Cs)
    ng = th.from_numpy(rng.integers(0, 40, C * Ns).astype(np.int64))
    h, r, t = ent[th.from_numpy(H)], rel[th.from_numpy(R)], ent[th.from_numpy(T_)]
    for neg_head in (False, True):
        pg, ngr = build_pos_graph(H, R, T_), NegGraph(ng, C, Cs, Ns, neg_head)
        pg.ndata["emb"], pg.edata["emb"] = ent[pg.ndata["id"]], rel[pg.edata["id"]]
        plain = KEModel.predict_neg_score(fake, pg, ngr)
        want = ko.negative_score(hp, ent[ng] if neg_head else h, r, t if neg_head else ent[ng], C, Cs, Ns, neg_head)
        assert th.equal(plain, want) and ngr.neg_sample_size == Ns
        got = KEModel.predict_neg_score(fake, pg, ngr, neg_deg_sample=True)
        assert ngr.neg_sample_size == Cs + Ns
        fbh = ko.Hyper(model="DistMult", hidden_dim=8, gamma=12.0, reg_coef=0.0, neg_deg_sample=True)
        fb = ko.forward_backward(fbh, ent, rel, pg.ndata["id"], *pg.all_edges(), pg.edata["id"], ng, C, Cs, Ns, neg_head)
        np.testing.assert_allclose(got.reshape(C * Cs, -1).numpy(), fb["neg_score"].numpy(), rtol=1e-6, atol=1e-7)
        # forward_test: rank = 1 + #{neg >= pos}
        logs = []
        ngr2 = NegGraph(ng, C, Cs, Ns, neg_head)
        KEModel.forward_test(fake, build_pos_graph(H, R, T_), ngr2, logs, -1)
        pos = ko.positive_score(hp, h, r, t)
        ranks = (want.reshape(C * Cs, -1) >= pos.reshape(-1, 1)).sum(1) + 1
        assert [l["MR"] for l in logs] == [float(x) for x in ranks.tolist()]
