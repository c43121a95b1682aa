"""Fused wgmma kernel (kge_fused.cu), stage by stage, against float64 evaluations of the reference formulas:

  stage 1  S = A.Bn^T (+ distance epilogue)        -> negative scores        (KGE_BUF_NEG_SCORE)
  stage 2  loss / softmax / backward coefficients   -> dL/dneg (/dist)        (kge_debug_set_dump, both passes)
  stage 3  G = V.Y with V as the register operand   -> negative / node grads  (KGE_BUF_NEG_GRAD, KGE_BUF_NODE_GRAD)

and the 5-launch fused step (kge_step_fused) against the oracle's step.  A failure message says which stage broke."""
import numpy as np
import pytest
import torch as th

import kge_oracle as ko
from test_gpu_parity import _random_step, _engine

pytestmark = pytest.mark.gpu

SHAPES = [  # (model, hidden, gamma, n_ent, n_rel, B, Cs, Ns, adv)
    ("TransE_l2", 400, 19.9, 14951, 1345, 1000, 200, 200, True),     # BASELINE configs[0/1] chunk shape
    ("DistMult", 400, 143.0, 5000, 100, 600, 200, 200, True),
    ("ComplEx", 400, 143.0, 5000, 100, 400, 200, 200, True),
    ("TransE_l2", 64, 10.0, 977, 13, 256, 64, 64, False),            # one 64-row tile, wide GEMM2 chunk, uniform weights
    ("TransE_l2", 96, 10.0, 977, 13, 320, 160, 72, True),            # ragged: Cs != Ns, two row tiles, D = 3 slab blocks
    ("DistMult", 40, 5.0, 500, 7, 96, 48, 24, True),                 # D not a multiple of 32
    ("TransE_l2", 400, 19.9, 14951, 1345, 6000, 200, 200, True),     # 60 tiles per pass
    ("DistMult", 128, 12.0, 3000, 20, 48000, 240, 240, True),        # 400 tiles > 132 SMs: persistent loop, ring hand-over between tiles
]


def _fp64_reference(hp, tables, si, C, Cs, Ns):
    t64 = [x.double().clone() for x in tables]
    ent, rel = t64[0], t64[2]
    nodes = ent[si["node_ids"]].clone().requires_grad_(True)
    rels = rel[si["rel_ids"]].clone().requires_grad_(True)
    negs = ent[si["neg_ids"]].clone().requires_grad_(True)
    h, t = nodes[si["head_local"]], nodes[si["tail_local"]]
    pos = ko.positive_score(hp, h, rels, t)
    if si["neg_head"]:
        neg = ko.negative_score(hp, negs, rels, t, C, Cs, Ns, True)
    else:
        neg = ko.negative_score(hp, h, rels, negs, C, Cs, Ns, False)
    neg = neg.reshape(-1, Ns)
    neg_leaf = neg.detach().clone().requires_grad_(True)
    loss, _ = ko.loss_terms(hp, pos.detach(), neg_leaf)
    loss.backward()
    g = neg_leaf.grad                                   # dL/dneg_ij
    if hp.model == "TransE_l2":
        g = g / (hp.gamma - neg.detach())               # the kernel carries dL/dneg / dist
    return neg.detach(), g


@pytest.mark.parametrize("cfg", SHAPES, ids=lambda c: "%s_d%d_B%d_%dx%d" % (c[0], c[1], c[5], c[6], c[7]))
@pytest.mark.parametrize("neg_head", [False, True])
def test_fused_kernel_stages(cfg, neg_head):
    from dglke_b200 import _lib
    model, hidden, gamma, n_ent, n_rel, B, Cs, Ns, adv = cfg
    hp = ko.Hyper(model=model, hidden_dim=hidden, gamma=gamma, lr=0.1, reg_coef=1e-6, reg_norm=3, adversarial=adv)
    ent, es, rel, rs = ko.init_tables(hp, n_ent, n_rel, seed=3)
    es.uniform_(0.0, 1e-3)
    rs.uniform_(0.0, 1e-3)
    si, C = _random_step(hp, n_ent, n_rel, B, Cs, Ns, neg_head, seed=31)
    S64, V64 = _fp64_reference(hp, (ent, es, rel, rs), si, C, Cs, Ns)
    eng, _ = _engine(hp, ent, es, rel, rs)
    dev = eng.device
    dump = th.full((2 * B * Ns,), float("nan"), dtype=th.float32, device=dev)
    eng.h.set_dump(dump)
    try:
        d = lambda t: t.to(dev)
        eng.forward_backward(d(si["node_ids"]), d(si["head_local"]), d(si["tail_local"]), d(si["rel_ids"]),
                             d(si["neg_ids"]), Cs, Ns, neg_head)
        S = eng.read(_lib.BUF_NEG_SCORE, (B, Ns)).double().cpu()
        th.cuda.synchronize()
        VP = dump[:B * Ns].reshape(B, Ns).double().cpu()
        VN = dump[B * Ns:].reshape(C, Ns, Cs).transpose(1, 2).reshape(B, Ns).double().cpu()
    finally:
        eng.h.set_dump(None)
    report = []

    def stage(name, got, want, rtol, atol_scale):
        err = (got - want).abs()
        scale = float(want.abs().max())
        bad = err > (rtol * want.abs() + atol_scale * scale)
        nan = int(th.isnan(got).sum())
        msg = "%s: max|err| %.3e (scale %.3e), bad %d / %d, nan %d" % (name, float(th.nan_to_num(err).max()), scale,
                                                                       int(bad.sum()), err.numel(), nan)
        if bad.any() or nan:
            idx = th.nonzero(bad | th.isnan(got))[:8].tolist()
            msg += ", first bad (row, col): %s" % idx
        report.append((bool(bad.any()) or nan > 0, msg))

    stage("stage 1 scores S", S, S64, 1e-5, 2e-6 * (1.0 + gamma / max(float(S64.abs().max()), 1e-30)))
    stage("stage 2 coefficients, positive-side pass", VP, V64, 2e-5, 2e-6)
    stage("stage 2 coefficients, negative-side pass", VN, V64, 2e-5, 2e-6)
    text = "\n".join(m for _, m in report)
    print(text)
    assert not any(b for b, _ in report), text


@pytest.mark.parametrize("cfg", SHAPES[:6], ids=lambda c: "%s_d%d_B%d_%dx%d" % (c[0], c[1], c[5], c[6], c[7]))
def test_fused_step_five_launches_matches_oracle(cfg):
    """kge_step_fused (prep, fused P, fused N, chain, cooperative update): tables and log scalars after 3 alternating
    steps against the oracle; exactly 5 kernel launches per step."""
    model, hidden, gamma, n_ent, n_rel, B, Cs, Ns, adv = cfg
    hp = ko.Hyper(model=model, hidden_dim=hidden, gamma=gamma, lr=0.1, reg_coef=1e-6, reg_norm=3, adversarial=adv)
    ent, es, rel, rs = ko.init_tables(hp, n_ent, n_rel, seed=4)
    es.uniform_(0.0, 1e-3)
    rs.uniform_(0.0, 1e-3)
    eng, (e, e_s, r, r_s) = _engine(hp, ent, es, rel, rs)
    dev = eng.device
    o = [x.clone() for x in (ent, es, rel, rs)]
    per_step = []
    for step in range(3):
        neg_head = step % 2 == 1
        si, C = _random_step(hp, n_ent, n_rel, B, Cs, Ns, neg_head, seed=200 + step)
        fb = ko.train_step(hp, o[0], o[1], o[2], o[3], si["node_ids"], si["head_local"], si["tail_local"],
                           si["rel_ids"], si["neg_ids"], C, Cs, Ns, neg_head)
        d = lambda t: t.to(dev)
        c0 = eng.h.launch_count()
        log4 = eng.step(d(si["node_ids"]), d(si["head_local"]), d(si["tail_local"]), d(si["rel_ids"]), d(si["neg_ids"]),
                        Cs, Ns, neg_head)
        per_step.append(eng.h.launch_count() - c0)
        got = log4.cpu().numpy()
        for i, k in enumerate(("pos_loss", "neg_loss", "loss", "regularization")):
            np.testing.assert_allclose(got[i], fb["log"][k], rtol=5e-5, atol=1e-9, err_msg="step %d %s" % (step, k))
    th.cuda.synchronize()
    for got, want, name in ((e, o[0], "entity table"), (e_s, o[1], "entity state"), (r, o[2], "relation table"),
                            (r_s, o[3], "relation state")):
        w = want.numpy()
        np.testing.assert_allclose(got.cpu().numpy(), w, rtol=1e-4, atol=5e-6 * float(np.abs(w).max()), err_msg=name)
    assert per_step[-1] <= 5, per_step


@pytest.mark.parametrize("model,hidden,de", [("TransE_l1", 64, False), ("RotatE", 32, True), ("RESCAL", 32, False),
                                             ("DistMult", 20, False)])
def test_step_fused_schedule_with_the_tile_kernels(model, hidden, de):
    """kge_step_fused on shapes / models the wgmma kernel does not take (L1, RotatE, RESCAL, D < 32): same fused-step
    schedule (no node cache, dense relation sums, log scalars from the update kernel) over the fp32 tile kernels."""
    hp = ko.Hyper(model=model, hidden_dim=hidden, gamma=8.0, lr=0.1, reg_coef=1e-6, reg_norm=3, adversarial=True,
                  double_ent=de)
    n_ent, n_rel, B, Cs, Ns = 700, 9, 96, 32, 24
    ent, es, rel, rs = ko.init_tables(hp, n_ent, n_rel, seed=6)
    es.uniform_(0.0, 1e-3)
    rs.uniform_(0.0, 1e-3)
    eng, (e, e_s, r, r_s) = _engine(hp, ent, es, rel, rs)
    o = [x.clone() for x in (ent, es, rel, rs)]
    for step in range(2):
        neg_head = step % 2 == 1
        si, C = _random_step(hp, n_ent, n_rel, B, Cs, Ns, neg_head, seed=300 + step)
        fb = ko.train_step(hp, o[0], o[1], o[2], o[3], si["node_ids"], si["head_local"], si["tail_local"],
                           si["rel_ids"], si["neg_ids"], C, Cs, Ns, neg_head)
        d = lambda t: t.to(eng.device)
        got = eng.step(d(si["node_ids"]), d(si["head_local"]), d(si["tail_local"]), d(si["rel_ids"]), d(si["neg_ids"]),
                       Cs, Ns, neg_head).cpu().numpy()
        for i, k in enumerate(("pos_loss", "neg_loss", "loss", "regularization")):
            np.testing.assert_allclose(got[i], fb["log"][k], rtol=5e-5, atol=1e-9, err_msg="step %d %s" % (step, k))
    th.cuda.synchronize()
    for got, want, name in ((e, o[0], "entity table"), (e_s, o[1], "entity state"), (r, o[2], "relation table"),
                            (r_s, o[3], "relation state")):
        w = want.numpy()
        np.testing.assert_allclose(got.cpu().numpy(), w, rtol=1e-4, atol=5e-6 * float(np.abs(w).max()), err_msg=name)


def test_fused_and_unfused_paths_agree():
    """Same step through the fused kernel and through the separate GEMM / loss kernels (kge_set_fused 0)."""
    from dglke_b200 import _lib
    hp = ko.Hyper(model="TransE_l2", hidden_dim=400, gamma=19.9, lr=0.25, reg_coef=1e-9, adversarial=True)
    res = []
    for mode in (1, 0):
        ent, es, rel, rs = ko.init_tables(hp, 14951, 1345, seed=0)
        eng, (e, e_s, r, r_s) = _engine(hp, ent, es, rel, rs)
        eng.h.set_fused(mode)
        try:
            si, C = _random_step(hp, 14951, 1345, 2000, 200, 200, False, seed=5)
            d = lambda t: t.to(eng.device)
            log4 = eng.step(d(si["node_ids"]), d(si["head_local"]), d(si["tail_local"]), d(si["rel_ids"]), d(si["neg_ids"]),
                            200, 200, False).cpu().numpy().copy()
            th.cuda.synchronize()
            res.append((log4, e.cpu().numpy().copy(), r.cpu().numpy().copy()))
        finally:
            eng.h.set_fused(-1)
    np.testing.assert_allclose(res[0][0], res[1][0], rtol=2e-5)
    np.testing.assert_allclose(res[0][1], res[1][1], rtol=1e-4, atol=1e-6)
    np.testing.assert_allclose(res[0][2], res[1][2], rtol=1e-4, atol=1e-6)


def test_fused_kernel_stress_200_runs():
    """200 back-to-back runs of the fused kernels on fresh random rows (hot chunk shape, both corruption modes): every
    run's scores and both coefficient passes against float64.  A race in the TMA / mbarrier / wgmma hand-offs would show
    up as sporadic garbage; this is the default engine's collected stress test (tests/stress_umma.py is the manual one
    for the stand-alone GEMMs)."""
    from dglke_b200 import _lib
    hp = ko.Hyper(model="TransE_l2", hidden_dim=400, gamma=19.9, lr=0.1, reg_coef=1e-9, adversarial=True)
    n_ent, n_rel, B, Cs, Ns = 3000, 11, 800, 200, 200
    g = th.Generator().manual_seed(123)
    bad = []
    eng = None
    dump = None
    for it in range(200):
        ent = (th.rand(n_ent, 400, generator=g) - 0.5) * 0.11
        rel = (th.rand(n_rel, 400, generator=g) - 0.5) * 0.11
        es, rs = th.zeros(n_ent), th.zeros(n_rel)
        neg_head = bool(it & 1)
        si, C = _random_step(hp, n_ent, n_rel, B, Cs, Ns, neg_head, seed=1000 + it)
        S64, V64 = _fp64_reference(hp, (ent, es, rel, rs), si, C, Cs, Ns)
        eng, _ = _engine(hp, ent, es, rel, rs)
        if dump is None:
            dump = th.empty(2 * B * Ns, dtype=th.float32, device=eng.device)
        dump.fill_(float("nan"))
        eng.h.set_dump(dump)
        try:
            d = lambda t: t.to(eng.device)
            eng.forward_backward(d(si["node_ids"]), d(si["head_local"]), d(si["tail_local"]), d(si["rel_ids"]),
                                 d(si["neg_ids"]), Cs, Ns, neg_head)
            S = eng.read(_lib.BUF_NEG_SCORE, (B, Ns)).double().cpu()
            VP = dump[:B * Ns].reshape(B, Ns).double().cpu()
            VN = dump[B * Ns:].reshape(C, Ns, Cs).transpose(1, 2).reshape(B, Ns).double().cpu()
        finally:
            eng.h.set_dump(None)
        eS = float(((S - S64).abs() / (1e-5 * S64.abs() + 2e-5)).max())
        eP = float(((VP - V64).abs() / (2e-5 * V64.abs() + 2e-6 * float(V64.abs().max()))).max())
        eN = float(((VN - V64).abs() / (2e-5 * V64.abs() + 2e-6 * float(V64.abs().max()))).max())
        if not (eS <= 1.0 and eP <= 1.0 and eN <= 1.0):        # also catches NaN
            bad.append((it, eS, eP, eN))
    assert not bad, "runs outside tolerance (iteration, score, coef P, coef N in units of the tolerance): %s" % bad[:10]
