"""The training step's increments -- Delta row = after - before and Delta state_sum -- against float64, from a state in
which every term of the update is visible.

A step's only outputs are the tables, their Adagrad state and the log scalars, so the update has to be judged from the
tables.  Compared whole, with the state the other hot-shape tests start from (U(0, 1e-3)), most of it cannot be seen:
at d = 400 a row's increment mean(g^2) is ~5e-7 of that state, far below any table tolerance, and with a zero state a
row that occurs once moves by -lr g / rms(g), whatever the scale of g.  Here every step starts from a state seeded out
of the float64 oracle:

  1. a float64 pre-pass (kge_oracle.forward_backward on the device's tables) gives every traced gradient; an entity
     row's increment m sums its node occurrence and all of its negative slots, a relation row's its edges;
  2. touched rows get state_sum = kappa * m, kappa log-uniform in [1/4, 4] (fixed seed); untouched rows a random state.
     Delta row then depends on the scale of g and on the state increment at order one;
  3. reg_coef (the case table's value) is the geometric mean, over the three trace entries, of the coefficient at
     which reg'(x) equals the loss gradient in the entry's median row;
  4. Delta row and Delta state are compared element by element with the float64 step from the same tables and state:

       |Delta_dev - Delta_64| <= sum over contributions of (lr beta / sigma + |Delta_c| dsigma / sigma) + n 1/2 ulp(x)
       |Dstate_dev - Dstate_64| <= 1e-4 Dstate_64 + n 1/2 ulp(state)

     beta = 5e-5 |g| + 1e-5 max|g_entry| is the gradient tolerance of test_gpu_parity, sigma = sqrt(s0 + m) + 1e-10
     the contribution's Adagrad denominator and dsigma what beta does to it through m; n counts the rounded adds that
     reach the element.  TransE_l1 adds, where a_k - b_k is within fp32 rounding of the kink of |.|, the change a
     flipped sign can make (_l1_kink_allowance), to beta and to the state bound.  Every case must stay within half of
     its bound (the largest fraction is printed), the log scalars within rtol 2e-5, and every row and state entry the
     step does not touch must be bit-identical.

test_visibility_of_every_term (no GPU) keeps this regime honest: for every case, dropping reg', dropping one entry's
state increment, scaling one entry's gradient by 1.01 or applying the negative entry before the node entry must move
the float64 reference by more than 4x the bound in at least 1 % of the rows concerned.

KGE_B200_NO_COOP and KGE_B200_NO_BULKRED are read once per process: tests/step_increments_env.py runs those cases in
a process of its own."""
import dataclasses
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch as th

import kge_oracle as ko
from test_gpu_parity import _random_step, _engine
from test_gpu_sharded import sharded, _engine as _sharded_engine, _deferred, _batch, _on_device  # noqa: F401

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LR = 0.1
RTOL_G, ATOL_G = 5e-5, 1e-5         # gradient tolerances of test_gpu_parity: rtol, atol as a fraction of the entry's max
RTOL_S = 1e-4                       # state increments
RTOL_LOG = 2e-5
USE = 0.5                           # the share of its bound a case may use
VISIBLE, VISIBLE_ROWS = 4.0, 0.01   # visibility guard: a change must exceed 4x the bound in >= 1 % of the rows concerned


@dataclasses.dataclass(frozen=True)
class Case:
    name: str
    model: str
    hidden: int
    gamma: float
    n_ent: int
    n_rel: int
    B: int
    Cs: int
    Ns: int
    reg_coef: float                 # from the rule of step 3 (test_visibility_of_every_term re-derives it)
    reg_norm: int = 3
    adv: bool = True
    de: bool = False
    dr: bool = None                 # double relation rows (default: as de)
    zipf: bool = False
    weighted: bool = False
    loss_genre: str = "Logsigmoid"
    pairwise: bool = False
    margin: float = 1.0

    def hyper(self):
        return ko.Hyper(model=self.model, hidden_dim=self.hidden, gamma=self.gamma, lr=LR, reg_coef=self.reg_coef,
                        reg_norm=self.reg_norm, adversarial=self.adv, adv_temperature=1.0, double_ent=self.de,
                        double_rel=self.de if self.dr is None else self.dr, loss_genre=self.loss_genre,
                        margin=self.margin, pairwise=self.pairwise)


BENCH = dict(model="TransE_l2", hidden=400, gamma=19.9, n_ent=14951, n_rel=1345, B=13200, Cs=200, Ns=200)
# kge_step_fused on the wgmma kernels
FUSED = [
    Case("TransE_l2_d400_bench", reg_coef=3.4e-4, **BENCH),                       # the benchmark's step, one wave
    Case("TransE_l2_d400_bench_zipf", reg_coef=3.5e-4, zipf=True, **BENCH),       # ids both positive node and negative
    Case("TransE_l2_d400_bench_norm1", reg_coef=1.4e-6, reg_norm=1, **BENCH),     # reg_grad_any in k_fused<N>
    Case("TransE_l2_d400_bench_norm2", reg_coef=2.2e-5, reg_norm=2, **BENCH),
    Case("DistMult_d400", "DistMult", 400, 143.0, 5000, 100, 600, 200, 200, reg_coef=4.4e-5),
    Case("ComplEx_d400", "ComplEx", 400, 143.0, 5000, 100, 600, 200, 200, reg_coef=6.6e-5, de=True),  # D = 800
    Case("TransE_l2_d512", "TransE_l2", 512, 19.9, 4999, 100, 1000, 200, 200, reg_coef=6.5e-3),  # widest bulk row
    Case("TransE_l2_d516", "TransE_l2", 516, 19.9, 4999, 100, 1000, 200, 200, reg_coef=6.6e-3),  # first row past it
    Case("TransE_l2_d128_240x240", "TransE_l2", 128, 10.0, 3000, 100, 960, 240, 240, reg_coef=2.8e-3),  # NV = 256
    Case("TransE_l2_d400_B1040_208x200", "TransE_l2", 400, 19.9, 14951, 1345, 1040, 208, 200, reg_coef=4.3e-3),
    Case("DistMult_d40", "DistMult", 40, 5.0, 500, 7, 96, 48, 24, reg_coef=4.3e-4),                 # D < one chunk
    Case("TransE_l2_d400_weighted", "TransE_l2", 400, 19.9, 14951, 1345, 1000, 200, 200, reg_coef=3.7e-3,
         weighted=True),
    Case("TransE_l2_d400_uniform", "TransE_l2", 400, 19.9, 14951, 1345, 1000, 200, 200, reg_coef=4.5e-3, adv=False),
]
# the fused schedule over the fp32 tile kernels
TILES = [
    Case("TransE_l1_d400", "TransE_l1", 400, 19.9, 3000, 50, 400, 200, 200, reg_coef=1.4e-1),
    Case("RotatE_d200_de", "RotatE", 200, 12.0, 5000, 53, 512, 256, 256, reg_coef=4.8e-2, de=True, dr=False),
    Case("RESCAL_d64", "RESCAL", 64, 12.0, 2000, 20, 128, 64, 64, reg_coef=1.0e-3, adv=False),
]
# kge_forward_backward + kge_update
THREE_CALL = [
    Case("TransE_l2_d400", "TransE_l2", 400, 19.9, 14951, 1345, 1000, 200, 200, reg_coef=4.5e-3),
    Case("RESCAL_d500", "RESCAL", 500, 12.0, 2000, 6, 128, 64, 64, reg_coef=1.9e-3, adv=False),
    Case("TransE_l2_d400_hinge_pw", "TransE_l2", 400, 19.9, 3000, 40, 400, 200, 200, reg_coef=2.1e-2, adv=False,
         loss_genre="Hinge", pairwise=True, margin=4.0),
]
HOST = Case("TransE_l2_d400_host", "TransE_l2", 400, 19.9, 14951, 1345, 1000, 200, 200, reg_coef=4.5e-3)
SHARDED = Case("TransE_l2_d400_2shards", "TransE_l2", 400, 19.9, 14951, 1345, 1000, 200, 200, reg_coef=4.5e-3)
ENV_CASES = [FUSED[0], FUSED[5]]
ALL = FUSED + TILES + THREE_CALL + [HOST, SHARDED]
_ids = lambda c: c.name


# ---------------------------------------------------------------------------------------------------- float64 side
def _steps(case, neg_head, seed):
    hp = case.hyper()
    si, C = _random_step(hp, case.n_ent, case.n_rel, case.B, case.Cs, case.Ns, neg_head, seed=seed, zipf=case.zipf)
    if case.weighted:
        si["edge_weight"] = th.from_numpy(np.random.default_rng(seed + 1).uniform(0.5, 1.5, case.B).astype(np.float32))
    return hp, si, C


def _prepass(hp, ent, rel, si, C, Cs, Ns, stale_ent=None):
    """float64 forward_backward on the given fp32 tables (the gradients do not depend on the state)"""
    w = si.get("edge_weight")
    read = ent if stale_ent is None else stale_ent
    fb = ko.forward_backward(hp, read.double(), rel.double(), si["node_ids"], si["head_local"], si["tail_local"],
                             si["rel_ids"], si["neg_ids"], C, Cs, Ns, si["neg_head"], None if w is None else w.double())
    if hp.model == "TransE_l1":
        fb["kink"] = _l1_kink_allowance(hp, read, rel, si, C, Cs, Ns)
    return fb


def _l1_kink_allowance(hp, ent, rel, si, C, Cs, Ns):
    """TransE_l1 differentiates |a_k - b_k| through sign(a_k - b_k), with a = h + r (t - r when the heads are corrupted)
    rounded to fp32 once.  Where a_k - b_k is within 4x that rounding of 0 the device's sign is not determined by the
    inputs, and the pair's coefficient V_ij may land on either side: a flip moves that element of the negative, the node
    and the relation gradient by 2 |V_ij|.  The allowance is twice that (every term of the bound is held to half).  The
    positive side must stay clear of its kink (asserted)."""
    e, r = ent.double(), rel.double()
    nh = si["neg_head"]
    h, t = e[si["node_ids"][si["head_local"]]], e[si["node_ids"][si["tail_local"]]]
    rr, ng = r[si["rel_ids"]], e[si["neg_ids"]]
    pos = hp.gamma - (h + rr - t).abs().sum(1)
    assert bool(((h + rr - t).abs() > 2.0 ** -22 * (h.abs() + rr.abs() + t.abs())).all()), "positive score on a kink"
    neg = (ko.negative_score(hp, ng, rr, t, C, Cs, Ns, True) if nh else
           ko.negative_score(hp, h, rr, ng, C, Cs, Ns, False)).reshape(-1, Ns).requires_grad_(True)
    w = si.get("edge_weight")
    loss, _ = ko.loss_terms(hp, pos, neg, None if w is None else w.double())
    V = th.autograd.grad(loss, neg)[0].abs().reshape(C, Cs, Ns, 1)
    a = (t - rr) if nh else (h + rr)
    tau = 2.0 ** -22 * (t.abs() + rr.abs()) if nh else 2.0 ** -22 * (h.abs() + rr.abs())
    D = a.shape[1]
    a, tau, b = a.reshape(C, Cs, 1, D), tau.reshape(C, Cs, 1, D), ng.reshape(C, 1, Ns, D)
    tie = ((a - b).abs() <= tau).double()
    allow_a = (4.0 * V * tie).sum(2).reshape(-1, D)
    allow_b = (4.0 * V * tie).sum(1).reshape(-1, D)
    own = si["tail_local"] if nh else si["head_local"]
    nodes = th.zeros(si["node_ids"].numel(), D, dtype=th.float64).index_add_(0, own, allow_a)
    return dict(nodes=nodes, negs=allow_b, rels=allow_a, ties=int(tie.sum()))


def _reg_prime(hp, x):
    p = hp.reg_norm
    return hp.reg_coef * p * x.abs().pow(p - 1) * x.sign()


def _entries(fb, si):
    return [("nodes", si["node_ids"], fb["nodes_grad"], fb["nodes"]), ("negs", si["neg_ids"], fb["negs_grad"], fb["negs"]),
            ("rels", si["rel_ids"], fb["rels_grad"], fb["rels"])]


def _reg_coef_rule(hp, fb, si):
    """geometric mean over the entries of the coefficient at which reg' equals the loss gradient in the median row"""
    rms = lambda g: g.pow(2).mean(1).sqrt()
    unit = dataclasses.replace(hp, reg_coef=1.0)
    logs = []
    for _, _, g, x in _entries(fb, si):
        loss_g = g - _reg_prime(hp, x)
        ratio = rms(loss_g) / rms(_reg_prime(unit, x)).clamp_min(1e-300)
        logs.append(math.log(float(ratio.median())))
    return math.exp(sum(logs) / len(logs)), [math.exp(v) for v in logs]


def _seed_states(fb, si, n_ent, n_rel, seed):
    """state_sum = kappa * m on touched rows (kappa log-uniform in [1/4, 4]), U(0, 2 median m) elsewhere (fp32)"""
    rng = np.random.default_rng(seed)
    out = []
    for n, parts in ((n_ent, [(si["node_ids"], fb["nodes_grad"]), (si["neg_ids"], fb["negs_grad"])]),
                     (n_rel, [(si["rel_ids"], fb["rels_grad"])])):
        m = th.zeros(n, dtype=th.float64)
        hit = th.zeros(n, dtype=th.bool)
        for idx, g in parts:
            m.index_add_(0, idx, g.pow(2).mean(1))
            hit[idx] = True
        kappa = np.exp(rng.uniform(math.log(0.25), math.log(4.0), n))
        med = float(m[hit].median())
        s = rng.uniform(0.0, 2.0 * med, n)
        s[hit.numpy()] = kappa[hit.numpy()] * m[hit].numpy()
        out.append(th.from_numpy(s.astype(np.float32)))
    return out


def _half_ulp(x):
    return 0.5 * np.spacing(np.abs(np.asarray(x, dtype=np.float64)).astype(np.float32)).astype(np.float64)


def _apply_entry(acc, idx, g, drop_state=False, kink=None):
    """one Adagrad trace entry into the float64 accumulators of one table, with its error bound (see module doc)"""
    beta = RTOL_G * g.abs() + ATOL_G * float(g.abs().max())
    if kink is not None:
        beta = beta + kink
        acc["dk"].index_add_(0, idx, (2.0 * g.abs() * kink + kink * kink).mean(1))
    m = g.pow(2).mean(1)
    dm = (2.0 * g.abs() * beta + beta * beta).mean(1)
    if not drop_state:
        acc["s"].index_add_(0, idx, m)
        acc["dm"].index_add_(0, idx, dm)
        acc["ns"].index_add_(0, idx, th.ones_like(m))
    s = acc["s"][idx]
    sig = s.sqrt() + 1e-10
    ulp_s = th.from_numpy(_half_ulp(s.numpy()))
    dsig = (acc["dm"][idx] + acc["ns"][idx] * ulp_s) / (2.0 * s.sqrt()).clamp_min(1e-300) + 2.0 ** -22 * sig
    d = -LR * g / sig.unsqueeze(1)
    acc["d"].index_add_(0, idx, d)
    acc["absd"].index_add_(0, idx, d.abs())
    acc["b"].index_add_(0, idx, LR * beta / sig.unsqueeze(1) + d.abs() * (dsig / sig).unsqueeze(1) + 2.0 ** -21 * d.abs())
    acc["nc"].index_add_(0, idx, th.ones_like(m))


def _reference(hp, emb, state, rel, rstate, fb, si, pert=None):
    """The float64 step from fp32 tables `emb, state, rel, rstate` with the gradients of `fb`.  Returns, per table,
    Delta row, Delta state and their bounds.  pert: a defect to apply (visibility guard)."""
    g = {k: gr.clone() for k, _, gr, _ in _entries(fb, si)}
    x = {k: xx for k, _, _, xx in _entries(fb, si)}
    if pert == "no_reg":
        for k in g:
            g[k] -= _reg_prime(hp, x[k])
    elif pert is not None and pert.startswith("scale_"):
        g[pert[6:]] *= 1.01
    res = {}
    for tab, e, s, order in (("ent", emb, state, ["nodes", "negs"]), ("rel", rel, rstate, ["rels"])):
        if pert == "neg_first" and tab == "ent":
            order = order[::-1]
        s0 = s.double()
        acc = dict(s=s0.clone(), dm=th.zeros_like(s0), dk=th.zeros_like(s0), ns=th.zeros_like(s0), nc=th.zeros_like(s0),
                   d=th.zeros(e.shape, dtype=th.float64), absd=th.zeros(e.shape, dtype=th.float64),
                   b=th.zeros(e.shape, dtype=th.float64))
        ids = dict(nodes=si["node_ids"], negs=si["neg_ids"], rels=si["rel_ids"])
        for k in order:
            _apply_entry(acc, ids[k], g[k], drop_state=(pert == "no_state_" + k), kink=fb["kink"][k] if "kink" in fb else None)
        big = e.double().abs() + acc["absd"]
        bound = acc["b"] + acc["nc"].unsqueeze(1) * th.from_numpy(_half_ulp(big.numpy()))
        ds = acc["s"] - s0
        sbound = RTOL_S * ds + acc["dk"] + (acc["ns"] + 1.0) * th.from_numpy(_half_ulp(acc["s"].numpy()))
        res[tab] = dict(d=acc["d"], b=bound, ds=ds, bs=sbound, hit=acc["nc"] > 0)
    return res


# ---------------------------------------------------------------------------------------------------- comparison
def _compare(what, ref, before, after):
    """`before` / `after`: (emb, state) fp32 CPU tensors of one table.  Returns the largest fraction of the bound used."""
    hit = ref["hit"]
    e0, s0 = before
    e1, s1 = after
    same = lambda a, b: th.equal(a.view(th.int32), b.view(th.int32))
    assert same(e0[~hit], e1[~hit]), "%s: a row the step does not touch changed" % what
    assert same(s0[~hit], s1[~hit]), "%s: a state entry the step does not touch changed" % what
    d = e1[hit].double() - e0[hit].double()
    fr = ((d - ref["d"][hit]).abs() / ref["b"][hit]).max(1).values
    ds = s1[hit].double() - s0[hit].double()
    frs = (ds - ref["ds"][hit]).abs() / ref["bs"][hit]
    assert not th.isnan(fr).any() and not th.isnan(frs).any(), "%s: NaN in the step's result" % what
    return float(fr.max()), float(frs.max())


def _check_log(hp, got, fb):
    worst = 0.0
    for i, k in enumerate(("pos_loss", "neg_loss", "loss", "regularization")):
        if k in fb["log"]:
            want = fb["log"][k]
            worst = max(worst, abs(float(got[i]) - want) / (RTOL_LOG * abs(want) + 1e-9))
    return worst


def _check_step(label, hp, before, after, fb, si, log=None, extra=None):
    """before / after: [emb, state, rel, rstate] fp32 CPU.  Asserts the bounds, prints the fractions used."""
    ref = _reference(hp, before[0], before[1], before[2], before[3], fb, si)
    fr = {}
    fr["ent rows"], fr["ent state"] = _compare(label + " entity table", ref["ent"], before[:2], after[:2])
    fr["rel rows"], fr["rel state"] = _compare(label + " relation table", ref["rel"], before[2:], after[2:])
    if log is not None:
        fr["log"] = _check_log(hp, log, fb)
    fr.update(extra or {})
    worst = max((k for k in fr if k != "log"), key=fr.get)
    print("%s: largest fraction of the bound %.3f (%s); %s" % (label, fr[worst], worst,
                                                                ", ".join("%s %.3f" % kv for kv in fr.items())))
    bad = {k: v for k, v in fr.items() if not v <= (1.0 if k == "log" else USE)}
    assert not bad, "%s: more than %.2f of the bound used (the log scalars: more than their tolerance): %s" % (
        label, USE, bad)


# ---------------------------------------------------------------------------------------------------- device side
def _seeded_engine(case, hp, si, C):
    """engine on the case's initial tables; returns the engine, its device tensors and the pre-pass"""
    ent, es, rel, rs = ko.init_tables(hp, case.n_ent, case.n_rel, seed=3)
    fb = _prepass(hp, ent, rel, si, C, case.Cs, case.Ns)
    es, rs = _seed_states(fb, si, case.n_ent, case.n_rel, seed=17)
    eng, dev_tabs = _engine(hp, ent, es, rel, rs)
    return eng, dev_tabs, fb


def _reseed(dev_tabs, hp, case, si, C, seed):
    """pre-pass on the device's current tables and state re-seeded in place (graph replays keep their pointers)"""
    e, es, r, rs = dev_tabs
    fb = _prepass(hp, e.cpu(), r.cpu(), si, C, case.Cs, case.Ns)
    s_e, s_r = _seed_states(fb, si, case.n_ent, case.n_rel, seed=seed)
    es.copy_(s_e)
    rs.copy_(s_r)
    th.cuda.synchronize()
    return fb


def _snap(dev_tabs):
    th.cuda.synchronize()
    return [x.cpu().clone() for x in dev_tabs]


def _dev(si):
    return {k: (v.cuda() if th.is_tensor(v) else v) for k, v in si.items()}


def run_fused_case(case, neg_head, label=None):
    """one kge_step_fused from a seeded state, checked (also the entry point of tests/step_increments_env.py)"""
    hp, si, C = _steps(case, neg_head, seed=41)
    eng, tabs, fb = _seeded_engine(case, hp, si, C)
    before = _snap(tabs)
    d = _dev(si)
    log = eng.step(d["node_ids"], d["head_local"], d["tail_local"], d["rel_ids"], d["neg_ids"], case.Cs, case.Ns, neg_head,
                   d["edge_weight"]).cpu().numpy()
    _check_step(label or "%s %s" % (case.name, "head" if neg_head else "tail"), hp, before, _snap(tabs), fb, si, log)


@pytest.mark.gpu
@pytest.mark.parametrize("case", FUSED + TILES, ids=_ids)
@pytest.mark.parametrize("neg_head", [False, True])
def test_fused_step_increments(case, neg_head):
    run_fused_case(case, neg_head)


@pytest.mark.gpu
@pytest.mark.parametrize("case", THREE_CALL, ids=_ids)
@pytest.mark.parametrize("neg_head", [False, True])
def test_three_call_increments(case, neg_head):
    """kge_forward_backward + kge_update: the non-fused update (per-edge relation entry, mean(g^2) of the negatives read
    back from their gradient rows)"""
    hp, si, C = _steps(case, neg_head, seed=43)
    eng, tabs, fb = _seeded_engine(case, hp, si, C)
    before = _snap(tabs)
    d = _dev(si)
    log = eng.forward_backward(d["node_ids"], d["head_local"], d["tail_local"], d["rel_ids"], d["neg_ids"], case.Cs,
                               case.Ns, neg_head, d["edge_weight"]).cpu().numpy()
    eng.update()
    _check_step("%s %s" % (case.name, "head" if neg_head else "tail"), hp, before, _snap(tabs), fb, si, log)


@pytest.mark.gpu
@pytest.mark.parametrize("pinned", [False, True])
def test_host_entry_point_increments(pinned):
    """kge_step_fused_host: pageable index arrays through the library's staging buffer, page-locked ones directly"""
    case = HOST
    for step, neg_head in enumerate((False, True)):
        hp, si, C = _steps(case, neg_head, seed=60 + step)
        if step == 0:
            eng, tabs, fb = _seeded_engine(case, hp, si, C)
        else:
            fb = _reseed(tabs, hp, case, si, C, seed=70 + step)
        before = _snap(tabs)
        hb = [si[k].pin_memory() if pinned else si[k] for k in ("node_ids", "head_local", "tail_local", "rel_ids", "neg_ids")]
        log = eng.step_host(*hb, case.Cs, case.Ns, neg_head)
        eng.sync()
        _check_step("host %s step %d" % ("pinned" if pinned else "pageable", step), hp, before, _snap(tabs), fb, si,
                    log.numpy().copy())


@pytest.mark.gpu
def test_graph_replay_increments():
    """bench.py's loop: warm-up steps, one CUDA graph per batch (with the edges' global endpoint ids), replays.  Three
    replays, the state re-seeded in place before each."""
    case = FUSED[0]
    hp, si0, C = _steps(case, False, seed=80)
    _, si1, _ = _steps(case, True, seed=81)
    eng, tabs, _ = _seeded_engine(case, hp, si0, C)
    dev = []
    for si in (si0, si1):
        d = _dev(si)
        d["head_ids"] = d["node_ids"][d["head_local"]].contiguous()
        d["tail_ids"] = d["node_ids"][d["tail_local"]].contiguous()
        dev.append(d)
    step = lambda d: eng.step(d["node_ids"], d["head_local"], d["tail_local"], d["rel_ids"], d["neg_ids"], case.Cs,
                              case.Ns, d["neg_head"], head_ids=d["head_ids"], tail_ids=d["tail_ids"])
    for d in dev:
        step(d)
    th.cuda.synchronize()
    graphs = []
    for d in dev:
        g = th.cuda.CUDAGraph()
        with th.cuda.graph(g):
            step(d)
        graphs.append(g)
    for k, b in enumerate((1, 0, 1)):
        si = (si0, si1)[b]
        fb = _reseed(tabs, hp, case, si, C, seed=90 + k)
        before = _snap(tabs)
        graphs[b].replay()
        log = eng.log4.cpu().numpy()
        _check_step("graph replay %d (%s)" % (k, "head" if b else "tail"), hp, before, _snap(tabs), fb, si, log)


@pytest.mark.gpu
def test_sharded_deferred_and_prefetched_increments(sharded):
    """2-shard entity table, deferred relation mode (ShardedTrainer.step with one rank): the caller's relation sums
    against float64 sum_e g_e and sum_e mean(g_e^2); entity increments through atomicAdd_system and the staged bulk
    reductions.  Step 0 announces step 1, whose fused kernels then read rows one step stale."""
    from dglke_b200 import _lib
    case = SHARDED
    hp = case.hyper()
    ent, es, rel, rs = ko.init_tables(hp, case.n_ent, case.n_rel, seed=3)
    tab = sharded(ent, es, 2)
    eng, r, r_s = _sharded_engine(hp, tab, rel, rs)
    rg, rgs = _deferred(eng, case.n_rel, hp.relation_dim)
    batches = [_batch(case.n_ent, case.n_rel, case.B, case.Cs, case.Ns, tab.boundary_ids(), 500 + s, s == 1)[0]
               for s in range(2)]
    C = case.B // case.Cs
    dev = [_on_device(si) for si in batches]
    stale = None
    for s, si in enumerate(batches):
        e0, _ = tab.read()
        fb = _prepass(hp, e0, r.cpu(), si, C, case.Cs, case.Ns, stale_ent=stale)
        s_e, s_r = _seed_states(fb, si, case.n_ent, case.n_rel, seed=510 + s)
        lo = 0
        for _, st_sh, rows in tab.allocs:
            st_sh[:rows].copy_(s_e[lo:lo + rows])
            lo += rows
        r_s.copy_(s_r)
        th.cuda.synchronize()
        before = [e0, tab.read()[1], r.cpu(), r_s.cpu()]
        d = dev[s]
        nxt = (dev[1]["node_ids"], dev[1]["neg_ids"]) if s == 0 else None
        eng.step_begin(d["node_ids"], d["head_local"], d["tail_local"], d["rel_ids"], d["neg_ids"], chunk_size=case.Cs,
                       neg_sample_size=case.Ns, neg_head=d["neg_head"], next_batch=nxt)
        log = eng.step_end().cpu().numpy()
        th.cuda.synchronize()
        # the caller's relation buffers before kge_rel_apply_dense consumes them
        got_rg = rg.view(case.n_rel, -1).cpu().double()
        got_rgs = rgs.cpu().double()
        g = fb["rels_grad"]
        beta = RTOL_G * g.abs() + ATOL_G * float(g.abs().max())
        n = th.zeros(case.n_rel, dtype=th.float64).index_add_(0, si["rel_ids"], th.ones(case.B, dtype=th.float64))
        want = th.zeros_like(got_rg).index_add_(0, si["rel_ids"], g)
        bnd = th.zeros_like(got_rg).index_add_(0, si["rel_ids"], beta)
        bnd += n.unsqueeze(1) * th.from_numpy(_half_ulp(th.zeros_like(got_rg).index_add_(0, si["rel_ids"], g.abs()).numpy()))
        want_s = th.zeros(case.n_rel, dtype=th.float64).index_add_(0, si["rel_ids"], g.pow(2).mean(1))
        bnd_s = RTOL_S * want_s + (n + 1.0) * th.from_numpy(_half_ulp(want_s.numpy()))
        hit = n > 0
        assert th.equal(got_rg[~hit], th.zeros_like(got_rg[~hit])) and th.equal(got_rgs[~hit], th.zeros_like(got_rgs[~hit])), \
            "step %d: relation sums written for a relation without edges" % s
        f_rg = float(((got_rg[hit] - want[hit]).abs() / bnd[hit]).max())
        f_rgs = float(((got_rgs[hit] - want_s[hit]).abs() / bnd_s[hit]).max())
        _lib.check(eng.lib.kge_rel_apply_dense(eng.h.raw, eng.rel.ref(), rg.data_ptr(), rgs.data_ptr(), float(hp.lr),
                                               eng.h.stream()))
        th.cuda.synchronize()
        e1, s1 = tab.read()
        _check_step("2 shards step %d%s" % (s, " (prefetched)" if s else ""), hp, before, [e1, s1, r.cpu(), r_s.cpu()],
                    fb, si, log, extra={"rel sums": f_rg, "rel state sums": f_rgs})
        stale = e0
    assert float(rgs.abs().max()) == 0.0 and float(rg.abs().max()) == 0.0, "relation sums not consumed"


@pytest.mark.gpu
@pytest.mark.parametrize("env", ["KGE_B200_NO_COOP", "KGE_B200_NO_BULKRED"])
def test_increments_under_environment_switch(env):
    """the three-launch k_update (KGE_B200_NO_COOP) and per-lane red.add instead of the bulk reductions
    (KGE_B200_NO_BULKRED), each in a process of its own: the switches are read once per process"""
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "step_increments_env.py")], capture_output=True,
                         text=True, timeout=900, cwd=ROOT, env={**os.environ, env: "1"})
    print(out.stdout)
    assert out.returncode == 0 and "STEP_INCREMENTS_ENV_OK" in out.stdout, out.stdout[-3000:] + out.stderr[-3000:]


# ---------------------------------------------------------------------------------------------------- no GPU
PERTURBATIONS = ["no_reg", "no_state_nodes", "no_state_negs", "no_state_rels", "scale_nodes", "scale_negs", "scale_rels",
                 "neg_first"]


@pytest.mark.parametrize("case", ALL, ids=_ids)
def test_visibility_of_every_term(case):
    """On the CPU, in float64: with the seeded state and the case's reg_coef, every term of the update moves the result
    by more than 4x the bound the GPU tests allow, in at least 1 % of the rows it concerns.  Also re-derives the case's
    reg_coef from its rule (within a factor 2, on either corruption side)."""
    for neg_head in (False, True):
        hp, si, C = _steps(case, neg_head, seed=41)
        ent, _, rel, _ = ko.init_tables(hp, case.n_ent, case.n_rel, seed=3)
        fb = _prepass(hp, ent, rel, si, C, case.Cs, case.Ns)
        coef, per_entry = _reg_coef_rule(hp, fb, si)
        assert 0.5 <= coef / case.reg_coef <= 2.0, "%s: the rule gives reg_coef %.3g, the table %.3g" % (
            case.name, coef, case.reg_coef)
        es, rs = _seed_states(fb, si, case.n_ent, case.n_rel, seed=17)
        ref = _reference(hp, ent, es, rel, rs, fb, si)
        rows = dict(nodes=si["node_ids"].unique(), negs=si["neg_ids"].unique())
        both = np.intersect1d(rows["nodes"].numpy(), rows["negs"].numpy())
        report = []
        for pert in PERTURBATIONS:
            alt = _reference(hp, ent, es, rel, rs, fb, si, pert)
            tab = "rel" if pert.endswith("rels") else "ent"
            if pert in ("no_reg",):
                concerned = [("ent", th.nonzero(ref["ent"]["hit"]).flatten()), ("rel", th.nonzero(ref["rel"]["hit"]).flatten())]
            elif pert == "neg_first":
                concerned = [("ent", th.from_numpy(both))]
            else:
                key = pert.split("_")[-1]
                concerned = [(tab, si["rel_ids"].unique() if key == "rels" else rows[key])]
            for t, idx in concerned:
                assert idx.numel() > 0, "%s %s: no rows concerned" % (case.name, pert)
                a, b = alt[t], ref[t]
                moved = th.maximum(((a["d"][idx] - b["d"][idx]).abs() / b["b"][idx]).max(1).values,
                                   (a["ds"][idx] - b["ds"][idx]).abs() / b["bs"][idx])
                share = float((moved > VISIBLE).double().mean())
                report.append("%s/%s %.2f" % (pert, t, share))
                assert share >= VISIBLE_ROWS, "%s %s: %s moves %.2f%% of the %s rows it concerns by more than %gx the bound" % (
                    case.name, "head" if neg_head else "tail", pert, 100 * share, t, VISIBLE)
        print("%s %s: reg_coef rule %.3g (per entry %s); share of rows moved: %s" % (
            case.name, "head" if neg_head else "tail", coef, ", ".join("%.3g" % v for v in per_entry), ", ".join(report)))
