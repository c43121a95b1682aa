"""Evaluation scoring against float64 at the shapes a real evaluation runs: kge_score_neg with one chunk per eval batch
and every entity (or a sample of 1 000) as candidates, kge_score_pos, score_func.infer, KEModel.forward_test ranks
and metrics, and training that resumes after an evaluation on the same handle.

The truth is kge_oracle's formulas (RESCAL's tail-mode quirk included) evaluated on float64 copies of the rows, in
blocks of candidates so that no intermediate exceeds BLOCK_BYTES.  Every device element must lie within
allowed_error() of it, a bound computed from the inputs alone; a case passes when its worst error uses at most half
of that bound.  Each case also checks, through the library's launch profiler, which kernel computed the scores."""
import ctypes
import math
import zlib

import numpy as np
import pytest
import torch as th

import kge_oracle as ko
from test_gpu_plugin import _args

pytestmark = pytest.mark.gpu

U = 2.0 ** -24                  # unit roundoff of fp32
C_SUM = 4.0                     # constant of the sqrt(D) term of allowed_error, fixed once for every model and route
BLOCK_BYTES = 256 << 20         # largest float64 intermediate of the reference
BILINEAR = ("DistMult", "ComplEx", "RESCAL")
GAMMA = {"TransE_l1": 19.9, "TransE_l2": 19.9, "DistMult": 143.0, "ComplEx": 143.0, "RESCAL": 12.0, "RotatE": 12.0}
WGMMA = "k_wgmma_gemm<score"
TILE = {"dot": "k_score<OP_DOT>", "l1": "k_score<OP_L1>", "rot": "k_rot_score"}


def allowed_error(model, D, gamma, s64, scale, s_dev=None):
    """Largest |device score - float64 score| an fp32 evaluation of the score may show, per element.

    `scale` is the error scale of the element, computed in float64 from the same rows:
      bilinear models   sum_k |a_k| |b_k|, with a the kept side as the formula builds it, evaluated on absolute values
                        (ComplEx: |er||rr| + |ei||ri| ...; RESCAL: |M_r| |p|), so that the rounding of a is covered too;
      TransE_l2         |a|^2 + |b|^2;
      TransE_l1, RotatE the distance, a sum of non-negative terms.

    Every score is a sum of D terms accumulated in fp32 (sequential FMAs or adds on the tiles, 3xTF32 wgmma steps on
    the tensor cores, where the dropped lo*lo term and the rounding of lo are each <= 2^-22 |a_k b_k|).  Its rounding
    error grows like sqrt(D) u sum|x_k| (Higham and Mary's probabilistic bound).  The worst case for it is a sum whose
    terms all have one sign (distances, |a|^2): D roundings, each within +-u of a partial sum that grows linearly, give
    a standard deviation of about sqrt(D)/3 u sum|x_k|, and the largest of the 10^7 elements of a case lies within 5.5
    of those, 1.8 sqrt(D) u sum|x_k|.  C_SUM = 4 is twice that, so that no case uses more than half of its bound.
    Terms of random sign (the bilinear scores) keep partial sums, and so errors, far smaller.

    The tensor cores round their fp32 accumulator toward zero, so the errors of the 3 ceil(D/8) accumulation steps of
    3xTF32 do not cancel: each is below 2^-23 of the accumulator.  When the terms share one sign -- a candidate close to
    the query's own row, a.b ~ |h|^2 -- the accumulator runs near the final dot product and the steps add up to
    3 ceil(D/8) 2^-23 |a.b|.  That term is added on every route (the fp32 tiles round to nearest and stay below it).

    Bilinear: C_SUM sqrt(D) u sum|a_k b_k| + 3 ceil(D/8) 2^-23 |s|, plus the rounding of a and of the stored result,
    <= 4u |s|.  Dropping one
    of the cross terms of 3xTF32 instead leaves an error of about 2^-11 sqrt(sum (a_k b_k)^2), roughly 2^-11/sqrt(D)
    sum|a_k b_k|: 2^9/D of the bound in a typical element (1.3x at D = 400, 0.3x at D = 1792), several times that in
    the worst of 10^5 elements.

    TransE_l2: the device and the reference both form d^2 = |a|^2 - 2 a.b + |b|^2, whose error is the same kind of sum,
    so |d_dev^2 - d64^2| <= C_SUM sqrt(D) u (|a|^2 + |b|^2) + 2 * 3 ceil(D/8) 2^-23 |a.b|, where
    a.b = (|a|^2 + |b|^2 - d64^2) / 2.  Since |d_dev - d64| = |d_dev^2 - d64^2| / (d_dev + d64),
    that turns into a bound on the distance exactly; without the device value, d_dev >= 0 gives <= delta/d64 and
    <= sqrt(delta).  sqrtf adds u d, the subtraction gamma - d one rounding of each operand, 2u (gamma + d).

    TransE_l1, RotatE: D non-negative terms, each exact to a few u of itself (|a_k| enters through the rounding of
    a = h + r or of the rotation, whose phase error is 2u |phase|), summed in fp32: C_SUM sqrt(D) u dist, plus 2u
    (gamma + dist) for gamma - dist.  RotatE's terms come from sqrt.approx.ftz.f32, bounded here by 4u of each term,
    4u dist in all (a bias need not cancel)."""
    k = C_SUM * U * math.sqrt(D)
    trunc = 3 * ((D + 7) // 8) * 2 * U
    if model in BILINEAR:
        return k * scale + (trunc + 4 * U) * s64.abs()
    if model == "TransE_l2":
        d64 = gamma - s64
        dd2 = k * scale + trunc * (scale - d64 * d64).abs()
        if s_dev is None:
            dd = th.minimum(dd2 / d64.clamp_min(1e-30), dd2.sqrt())
        else:
            dd = dd2 / (d64 + (gamma - s_dev).clamp_min(0.0)).clamp_min(1e-30)
        return dd + U * d64 + 2 * U * (gamma + d64)
    tol = k * scale + 2 * U * (gamma + scale)
    if model == "RotatE":
        tol = tol + 4 * U * scale
    return tol


# ---------------------------------------------------------------------------------------------------- float64 reference
def _hypers(model, hidden):
    """(kge_oracle.Hyper, engine.Hyper) of one model; ComplEx and RotatE take the reference recipes' -de (-dr)."""
    from dglke_b200.engine import Hyper
    kw = dict(model=model, hidden_dim=hidden, gamma=GAMMA[model], double_ent=model in ("ComplEx", "RotatE"),
              double_rel=model == "ComplEx")
    return ko.Hyper(**kw), Hyper(**kw)


def _seed(*parts):
    return zlib.crc32(repr(parts).encode())


def _tables(hp, n_ent, n_rel, kind, seed):
    """ko.init_tables, or a 'trained-like' variant: rows scaled by per-row factors in [0.5, 4] and relation entries up
    to +-3 emb_init (RotatE phases up to +-3 pi, score magnitudes spread out)."""
    ent, _, rel, _ = ko.init_tables(hp, n_ent, n_rel, seed=seed)
    if kind == "trained":
        g = th.Generator().manual_seed(seed + 1)
        ent *= th.empty(n_ent, 1).uniform_(0.5, 4.0, generator=g)
        rel = th.empty_like(rel).uniform_(-3 * hp.emb_init, 3 * hp.emb_init, generator=g)
    return ent, rel


def _kept_side(hp, p, r, neg_head):
    """Per positive row: the absolute-value form of the kept side (bilinear) or |a|^2 (TransE_l2), float64."""
    m, D = hp.model, p.shape[1]
    if m == "DistMult":
        return (p * r).abs()
    if m == "ComplEx":
        er, ei, rr, ri = p[:, :D // 2].abs(), p[:, D // 2:].abs(), r[:, :D // 2].abs(), r[:, D // 2:].abs()
        return th.cat((er * rr + ei * ri, er * ri + ei * rr), 1)
    if m == "RESCAL":
        return th.bmm(r.view(-1, D, D).abs(), p.abs().unsqueeze(-1)).squeeze(-1)
    if m == "TransE_l2":
        a = p - r if neg_head else p + r
        return (a * a).sum(1)
    return None


def _ref_blocks(hp, pos_e, rels, negs, C, Cs, Ns, neg_head):
    """Yields (chunk, first candidate, float64 scores [Cs, n], error scales [Cs, n]) over blocks of candidates.
    pos_e / rels: the positives' kept-side rows and relation rows [C*Cs, .]; negs: the candidates [C*Ns, D]."""
    D = pos_e.shape[1]
    per_cand = Cs * D * 48 if hp.model in ("TransE_l1", "RotatE") else Cs * 48 + D * 16
    nb = max(8, BLOCK_BYTES // per_cand)
    for c in range(C):
        p = pos_e[c * Cs:(c + 1) * Cs].double()
        r = rels[c * Cs:(c + 1) * Cs].double()
        kept = _kept_side(hp, p, r, neg_head)
        for j0 in range(0, Ns, nb):
            b = negs[c * Ns + j0:c * Ns + min(Ns, j0 + nb)].double()
            s = ko.negative_score(hp, *((b, r, p) if neg_head else (p, r, b)), 1, Cs, b.shape[0], neg_head)[0]
            if hp.model in BILINEAR:
                scale = kept @ b.abs().T
            elif hp.model == "TransE_l2":
                scale = kept[:, None] + (b * b).sum(1)[None, :]
            else:
                scale = hp.gamma - s
            yield c, j0, s, scale


def _pos_ref(hp, h, r, t, rows=8192):
    """float64 positive scores and their error scales, in blocks of rows."""
    out_s, out_scale = [], []
    D = h.shape[1]
    for i in range(0, h.shape[0], rows):
        hh, rr, tt = (x[i:i + rows].double() for x in (h, r, t))
        s = ko.positive_score(hp, hh, rr, tt)
        if hp.model == "DistMult":
            scale = (hh * rr * tt).abs().sum(1)
        elif hp.model == "ComplEx":
            hr, hi, tr, ti, r_, ri = (x.abs() for x in (hh[:, :D // 2], hh[:, D // 2:], tt[:, :D // 2], tt[:, D // 2:],
                                                        rr[:, :D // 2], rr[:, D // 2:]))
            scale = (hr * tr * r_ + hi * ti * r_ + hr * ti * ri + hi * tr * ri).sum(1)
        elif hp.model == "RESCAL":
            scale = (hh.abs() * th.bmm(rr.view(-1, D, D).abs(), tt.abs().unsqueeze(-1)).squeeze(-1)).sum(1)
        elif hp.model == "TransE_l2":
            a = hh + rr
            scale = (a * a).sum(1) + (tt * tt).sum(1)
        else:
            scale = hp.gamma - s
        out_s.append(s)
        out_scale.append(scale)
    return th.cat(out_s), th.cat(out_scale)


class _Worst:
    """Worst error-to-bound ratio over the compared elements (NaN or inf on the device counts as infinite)."""

    def __init__(self):
        self.ratio, self.where, self.n = 0.0, "", 0

    def add(self, got, want, tol, label=""):
        ratio = (got - want).abs() / tol
        ratio = th.where(th.isfinite(ratio), ratio, th.full_like(ratio, float("inf")))
        self.n += ratio.numel()
        i = int(ratio.argmax())
        if float(ratio.view(-1)[i]) >= self.ratio:
            self.ratio = float(ratio.view(-1)[i])
            idx = np.unravel_index(i, tuple(ratio.shape))
            self.where = "%s%s: device %.9g, float64 %.9g, bound %.3g" % (
                label, tuple(int(x) for x in idx), float(got[idx]), float(want[idx]), float(tol[idx]))

    def report(self, name):
        line = "%s: worst |err|/bound = %.3f over %d elements (at %s)" % (name, self.ratio, self.n, self.where)
        print(line)
        return line


def _score_neg(ehp, heads, rels, tails, C, Cs, Ns, neg_head):
    """kge_score_neg into an output that starts as NaN, so that an element the kernels never write cannot pass."""
    from dglke_b200 import _lib
    from dglke_b200.engine import _cfg_for
    h = _lib.get_handle(heads.device.index)
    cfg = _cfg_for(ehp, C * Cs, Cs, Ns, neg_head)
    out = th.full((C, Cs, Ns), float("nan"), dtype=th.float32, device=heads.device)
    heads, rels, tails = heads.contiguous(), rels.contiguous(), tails.contiguous()
    _lib.check(h.lib.kge_score_neg(h.raw, ctypes.byref(cfg), heads.data_ptr(), rels.data_ptr(), tails.data_ptr(),
                                   out.data_ptr(), h.stream()))
    return out


def _score_routes(h):
    """Score kernels launched since profiling was switched on: 'wgmma' and/or tile kernel names."""
    names = [n for n, _ in h.profile_read()]
    return {("wgmma" if n.startswith(WGMMA) else n) for n in names if n.startswith(WGMMA) or n in TILE.values()}


def _expect_route(routes, route, what):
    want = {"wgmma" if route == "wgmma" else TILE[route]}
    assert routes == want, "%s: scores computed by %s, expected %s" % (what, sorted(routes), sorted(want))


@pytest.fixture
def handle():
    """The shared handle of device 0, given back with the default engine and the profiler off."""
    from dglke_b200 import _lib
    h = _lib.get_handle(0)
    yield h
    h.profile_enable(False)
    h.set_engine(-1)


# ------------------------------------------------------------------------------------ kge_score_neg at evaluation shapes
SCORE_CASES = [  # (name, model, hidden, C, Cs, Ns, route, engine)
    ("DistMult400_16x14952", "DistMult", 400, 1, 16, 14952, "wgmma", -1),        # N tail 104, K tail 16
    ("DistMult400_16x14951", "DistMult", 400, 1, 16, 14951, "dot", -1),          # odd Ns, 64-wide tile tail
    ("TransE_l2_400_1000x14952", "TransE_l2", 400, 1, 1000, 14952, "wgmma", -1),  # 8 M tiles, last 104 rows; a2/b2
    ("TransE_l2_400_11x14952", "TransE_l2", 400, 1, 11, 14952, "dot", -1),       # the short last eval batch
    ("TransE_l2_400_3x12x5000", "TransE_l2", 400, 3, 12, 5000, "dot", -1),       # a2 / b2 taken per chunk
    ("ComplEx400de_3x16x4096", "ComplEx", 400, 3, 16, 4096, "wgmma", -1),        # D = 800, grid z = 3, exact N tiles
    ("DistMult32_8x8", "DistMult", 32, 1, 8, 8, "wgmma", -1),                    # smallest legal shape
    ("DistMult32_8x136", "DistMult", 32, 1, 8, 136, "wgmma", -1),                # one 128-tile overhanging M and N
    ("DistMult1792_16x14952", "DistMult", 1792, 1, 16, 14952, "wgmma", -1),      # largest D whose prep staging fits
    ("DistMult1800_16x14952", "DistMult", 1800, 1, 16, 14952, "dot", -1),        # first D beyond it
    ("RESCAL64_16x14951", "RESCAL", 64, 1, 16, 14951, "dot", -1),                # RESCAL scores always on the tiles
    ("RESCAL64_16x5000", "RESCAL", 64, 1, 16, 5000, "dot", -1),
    ("RESCAL200_16x14951", "RESCAL", 200, 1, 16, 14951, "dot", -1),
    ("RESCAL200_16x5000", "RESCAL", 200, 1, 16, 5000, "dot", -1),
    ("RotatE200de_16x14951", "RotatE", 200, 1, 16, 14951, "rot", -1),            # D = 400, phases beyond +-pi
    ("TransE_l1_400_3x16x5000", "TransE_l1", 400, 3, 16, 5000, "l1", -1),
    ("DistMult400_16x14952_engine0", "DistMult", 400, 1, 16, 14952, "dot", 0),   # the same inputs on the other engine
    ("TransE_l2_400_1000x14952_engine0", "TransE_l2", 400, 1, 1000, 14952, "dot", 0),
    ("TransE_l2_400_3x12x5000_engine0", "TransE_l2", 400, 3, 12, 5000, "dot", 0),
]


@pytest.mark.parametrize("tables", ["init", "trained"])
@pytest.mark.parametrize("case", SCORE_CASES, ids=lambda c: c[0])
def test_score_neg_at_eval_shapes(handle, case, tables):
    name, model, hidden, C, Cs, Ns, route, engine = case
    khp, ehp = _hypers(model, hidden)
    n_rel = 50
    seed = _seed(name.replace("_engine0", ""), tables)          # the engine-0 rows reuse their case's inputs
    ent, rel = _tables(khp, C * Ns, n_rel, tables, seed)         # candidates: every row of the table, chunk-major
    rng = np.random.default_rng(seed)
    pos_e = ent[th.from_numpy(rng.integers(0, C * Ns, C * Cs))]
    rels = rel[th.from_numpy(rng.integers(0, n_rel, C * Cs))]
    dev = th.device("cuda", 0)
    d_pos, d_rel, d_ent = pos_e.to(dev), rels.to(dev), ent.to(dev)
    handle.set_engine(engine)
    lines = []
    for neg_head in (False, True):
        handle.profile_enable(True)
        out = _score_neg(ehp, *((d_ent, d_rel, d_pos) if neg_head else (d_pos, d_rel, d_ent)), C, Cs, Ns, neg_head)
        _expect_route(_score_routes(handle), route, name)
        handle.profile_enable(False)
        got = out.cpu().double()
        worst = _Worst()
        for c, j0, s64, scale in _ref_blocks(khp, pos_e, rels, ent, C, Cs, Ns, neg_head):
            g = got[c, :, j0:j0 + s64.shape[1]]
            worst.add(g, s64, allowed_error(model, khp.entity_dim, khp.gamma, s64, scale, g), "chunk %d col+%d " % (c, j0))
        lines.append((worst.ratio, worst.report("%s %s neg_head=%s" % (name, tables, neg_head))))
    bad = [l for r, l in lines if not r <= 0.5]
    assert not bad, "\n".join(bad)


# ------------------------------------------------------------------------------------------- kge_score_pos and infer
POS_MODELS = [("TransE_l1", 400), ("TransE_l2", 400), ("DistMult", 400), ("ComplEx", 200), ("RESCAL", 32), ("RotatE", 200)]


@pytest.mark.parametrize("tables", ["init", "trained"])
@pytest.mark.parametrize("model,hidden", POS_MODELS)
def test_score_pos_65539_edges(model, hidden, tables):
    """65 539 edges: a tail in the one-warp-per-edge grid of the dense prep kernels."""
    from dglke_b200.engine import score_pos
    khp, ehp = _hypers(model, hidden)
    n, n_ent, n_rel = 65539, 5000, 40
    seed = _seed("pos", model, tables)
    ent, rel = _tables(khp, n_ent, n_rel, tables, seed)
    rng = np.random.default_rng(seed)
    h, t = (ent[th.from_numpy(rng.integers(0, n_ent, n))] for _ in range(2))
    r = rel[th.from_numpy(rng.integers(0, n_rel, n))]
    dev = th.device("cuda", 0)
    got = score_pos(ehp, h.to(dev), r.to(dev), t.to(dev)).cpu().double()
    s64, scale = _pos_ref(khp, h, r, t)
    worst = _Worst()
    worst.add(got, s64, allowed_error(model, khp.entity_dim, khp.gamma, s64, scale, got))
    line = worst.report("score_pos %s d=%d %s n=%d" % (model, khp.entity_dim, tables, n))
    assert worst.ratio <= 0.5, line


@pytest.mark.parametrize("model,hidden,route", [("RESCAL", 64, "dot"), ("TransE_l2", 400, "wgmma")])
def test_infer_8_heads_4_relations_4096_tails(handle, model, hidden, route):
    """score_func.infer: RESCAL through its own head-mode route (score_fun.py), TransE_l2 through the generic one."""
    from dglke_b200.general_models import KEModel
    khp, _ = _hypers(model, hidden)
    ent, rel = _tables(khp, 5000, 10, "trained", _seed("infer", model))
    m = KEModel(_args(), model, 5000, 10, hidden, khp.gamma)
    m.entity_emb.emb.copy_(ent)
    m.relation_emb.emb.copy_(rel)
    h, r, t = ent[:8], rel[:4], ent[100:4196]
    handle.profile_enable(True)
    got = m.score_func.infer(m.entity_emb.emb[:8], m.relation_emb.emb[:4], m.entity_emb.emb[100:4196]).cpu().double()
    _expect_route(_score_routes(handle), route, "infer %s" % model)
    handle.profile_enable(False)
    assert tuple(got.shape) == (8, 4, 4096)
    h, r, t = h.double(), r.double(), t.double()
    D = khp.entity_dim
    if model == "RESCAL":      # the edge score h^T M_r t (positive_score) of every combination
        M = r.view(4, D, D)
        s64 = th.einsum("id,jde,ke->ijk", h, M, t)
        scale = th.einsum("id,jde,ke->ijk", h.abs(), M.abs(), t.abs())
    else:
        hh, rr = h.repeat_interleave(4, 0), r.repeat(8, 1)             # row 4 i + j: (head i, relation j)
        s64 = ko.negative_score(khp, hh, rr, t, 1, 32, 4096, False).reshape(8, 4, 4096)
        a = hh + rr
        scale = ((a * a).sum(1)[:, None] + (t * t).sum(1)[None, :]).reshape(8, 4, 4096)
    worst = _Worst()
    worst.add(got, s64, allowed_error(model, D, khp.gamma, s64, scale, got))
    line = worst.report("infer %s d=%d 8x4x4096" % (model, D))
    assert worst.ratio <= 0.5, line


# ----------------------------------------------------------------------------------- forward_test at full-entity counts
N_REL = 20


def _planted(hp, n_ent, n_test, seed):
    """Tables plus n_test triples, every third planted to rank near the top: t ~ h + r (TransE_l2) or t leaning on
    h * r (DistMult), with a per-triple strength so that the ranks spread over 1 .. a few dozen."""
    ent, rel = _tables(hp, n_ent, N_REL, "init", seed)
    rng = np.random.default_rng(seed)
    H, R = rng.integers(0, n_ent // 2, n_test), rng.integers(0, N_REL, n_test)
    T = rng.integers(0, n_ent, n_test)
    planted = np.arange(0, n_test, 3)
    T[planted] = rng.choice(np.arange(n_ent // 2, n_ent), len(planted), replace=False)
    g = th.Generator().manual_seed(seed)
    for i in planted:
        h, r = ent[H[i]], rel[R[i]]
        if hp.model == "TransE_l2":
            ent[T[i]] = h + r + th.randn(h.shape, generator=g) * hp.emb_init * float(rng.uniform(0.75, 0.92))
        else:
            hr = h * r
            lam = float(rng.uniform(0.1, 0.3))
            ent[T[i]] = lam * hr / hr.norm() * ent[T[i]].norm() + (1 - lam) * ent[T[i]]
    return ent, rel, (H, R, T), planted


def _known_triples(H, R, T, n_ent, seed):
    """The positives plus triples sharing (head, relation) or (tail, relation) with them, and random ones."""
    rng = np.random.default_rng(seed)
    n = len(H)
    pick = rng.integers(0, n, 600)
    kh = np.concatenate([H, H[pick[:300]], rng.integers(0, n_ent, 300), rng.integers(0, n_ent, 1000)])
    kr = np.concatenate([R, R[pick[:300]], R[pick[300:]], rng.integers(0, N_REL, 1000)])
    kt = np.concatenate([T, rng.integers(0, n_ent, 300), T[pick[300:]], rng.integers(0, n_ent, 1000)])
    return kh, kr, kt


def _filter_mask(kh, kr, kt, h, r, t, cand, neg_head):
    """[len(h), len(cand)] True where the candidate makes a known triple (computed from sets, not TripleFilter)."""
    known = {}
    for a, b, c in zip(kh.tolist(), kr.tolist(), kt.tolist()):
        key = (c, b) if neg_head else (a, b)
        known.setdefault(key, set()).add(a if neg_head else c)
    col = {int(e): j for j, e in enumerate(cand)}
    mask = th.zeros(len(h), len(cand), dtype=th.bool)
    for i in range(len(h)):
        for e in known.get((int(t[i]), int(r[i])) if neg_head else (int(h[i]), int(r[i])), ()):
            if e in col:
                mask[i, col[e]] = True
    return mask


def _rank_intervals(hp, ent, rel, h, r, t, cand, neg_head, mask):
    """Near-tie interval of each positive's rank: [1 + #{neg > pos + tau}, 1 + #{neg >= pos - tau}], filtered
    candidates left out, tau = the two elements' allowed errors."""
    D = hp.entity_dim
    H, R, T = (th.from_numpy(np.asarray(x)) for x in (h, r, t))
    hr, rr, tr = ent[H], rel[R], ent[T]
    pos64, pscale = _pos_ref(hp, hr, rr, tr)
    ptol = allowed_error(hp.model, D, hp.gamma, pos64, pscale)
    cand_rows = ent[th.from_numpy(cand)]
    lo = th.ones(len(h), dtype=th.long)
    hi = th.ones(len(h), dtype=th.long)
    for _, j0, s64, scale in _ref_blocks(hp, tr if neg_head else hr, rr, cand_rows, 1, len(h), len(cand), neg_head):
        tau = allowed_error(hp.model, D, hp.gamma, s64, scale) + ptol[:, None]
        keep = ~mask[:, j0:j0 + s64.shape[1]] if mask is not None else th.ones_like(s64, dtype=th.bool)
        lo += ((s64 > pos64[:, None] + tau) & keep).sum(1)
        hi += ((s64 >= pos64[:, None] - tau) & keep).sum(1)
    return lo, hi


def _run_forward_test(handle, model, n_ent, filtered, n_cand=None, n_test=203, batch=16):
    from dglke_b200.general_models import KEModel
    from dglke_b200.graph import eval_batches, TripleFilter
    khp, _ = _hypers(model, 400)
    seed = _seed("ft", model, n_ent)
    ent, rel, (H, R, T), planted = _planted(khp, n_ent, n_test, seed)
    m = KEModel(_args(eval_filter=filtered), model, n_ent, N_REL, 400, khp.gamma)
    m.entity_emb.emb.copy_(ent)
    m.relation_emb.emb.copy_(rel)
    rng = np.random.default_rng(seed + 1)
    cand = np.arange(n_ent) if n_cand is None else np.sort(rng.choice(n_ent, n_cand, replace=False))
    kh, kr, kt = _known_triples(H, R, T, n_ent, seed + 2)
    known = TripleFilter(kh, kr, kt, N_REL) if filtered else None
    report = []
    for neg_head in (False, True):
        logs, want_routes, got_routes = [], [], []
        for pg, ng in eval_batches(H, R, T, n_ent, batch, neg_head, None if n_cand is None else cand, known):
            handle.profile_enable(True)
            m.forward_test(pg, ng, logs, 0)
            got_routes.append(_score_routes(handle))
            handle.profile_enable(False)
            nb = pg.number_of_edges()
            want_routes.append({"wgmma" if nb % 8 == 0 and len(cand) % 8 == 0 else TILE["dot"]})
        assert got_routes == want_routes, (got_routes, want_routes)
        mask = _filter_mask(kh, kr, kt, H, R, T, cand, neg_head) if filtered else None
        lo, hi = _rank_intervals(khp, ent, rel, H, R, T, cand, neg_head, mask)
        got = th.tensor([int(l["MR"]) for l in logs])
        out = ((got < lo) | (got > hi)).nonzero().view(-1).tolist()
        what = "%s n_ent=%d cand=%d %s neg_head=%s" % (model, n_ent, len(cand), "filtered" if filtered else "raw",
                                                      neg_head)
        assert not out, "%s: ranks outside their near-tie interval at %s: got %s, interval %s" % (
            what, out[:8], got[out[:8]].tolist(), list(zip(lo[out[:8]].tolist(), hi[out[:8]].tolist())))
        # the metrics the library reports, within what the intervals allow
        mean = lambda key: float(np.mean([l[key] for l in logs]))
        lo_f, hi_f = lo.double(), hi.double()
        bounds = {"MRR": ((1 / hi_f).mean(), (1 / lo_f).mean()), "MR": (lo_f.mean(), hi_f.mean())}
        for k in (1, 3, 10):
            bounds["HITS@%d" % k] = ((hi <= k).double().mean(), (lo <= k).double().mean())
        for key, (a, b) in bounds.items():
            assert float(a) - 1e-12 <= mean(key) <= float(b) + 1e-12, (what, key, mean(key), float(a), float(b))
        ties = int((hi > lo).sum())
        report.append("%s: MRR %.4f HITS@1 %.3f HITS@10 %.3f, planted median rank %d, %d of %d ranks with near-ties"
                      % (what, mean("MRR"), mean("HITS@1"), mean("HITS@10"), int(got[planted].median()), ties, len(got)))
        assert int(got[planted].median()) <= 10, report[-1]     # the planted triples do rank near the top
    print("\n".join(report))


@pytest.mark.parametrize("filtered", [False, True], ids=["raw", "filtered"])
@pytest.mark.parametrize("model,n_ent", [("TransE_l2", 14952), ("TransE_l2", 14951), ("DistMult", 14952),
                                         ("DistMult", 14951)])
def test_forward_test_ranks_full_entities(handle, model, n_ent, filtered):
    """203 triples in eval batches of 16: 12 full batches and one of 11.  With 14 952 entities the full batches take the
    wgmma engine and the last one the tiles, inside one evaluation; with 14 951 every batch takes the tiles."""
    _run_forward_test(handle, model, n_ent, filtered)


@pytest.mark.parametrize("filtered", [False, True], ids=["raw", "filtered"])
def test_forward_test_ranks_sampled_candidates(handle, filtered):
    """--neg_sample_size_eval: 1 000 sampled candidates per query."""
    _run_forward_test(handle, "TransE_l2", 14952, filtered, n_cand=1000)


# ------------------------------------------------------------------------- training after an evaluation on one handle
@pytest.fixture
def fresh_handle():
    """A handle of its own for device 0 (so that its step workspace starts empty), installed as the shared one for the
    duration of the test."""
    from dglke_b200 import _lib
    old = _lib._handles.get(0)
    h = _lib.Handle(0)
    _lib._handles[0] = h
    try:
        yield h
    finally:
        th.cuda.synchronize()
        if old is None:
            _lib._handles.pop(0, None)
        else:
            _lib._handles[0] = old
        h.close()


TRAIN_EVAL = [  # (model, n_ent, device sampler): the evaluation's workspace vs the training step's
    ("TransE_l2", 2001, True),      # (a) smaller, tiles: the evaluation writes over the node-gradient region
    ("TransE_l2", 2001, False),     # (a) the same on the 3-call path (host-sampled batches)
    ("TransE_l2", 14952, True),     # (b) larger: the arena is regrown
]


@pytest.mark.parametrize("model,n_ent,device_sampler", TRAIN_EVAL, ids=["a_fused", "a_three_call", "b_regrown"])
def test_training_resumes_correctly_after_an_evaluation(fresh_handle, model, n_ent, device_sampler):
    """What `train.py --valid` does: 3 training steps, a full forward_test evaluation, 3 more steps.  The tables must
    match the oracle (in float64) driven with the same batches and no evaluation."""
    from dglke_b200.general_models import KEModel
    from dglke_b200.graph import TripleSampler, eval_batches
    from dglke_b200.train import DeviceGraphSampler
    n_rel, B, N, lr, reg = 50, 1000, 200, 0.1, 1e-6
    rng = np.random.default_rng(_seed("train", model, n_ent))
    tr = [rng.integers(0, n_ent, 20000), rng.integers(0, n_rel, 20000), rng.integers(0, n_ent, 20000)]
    va = [rng.integers(0, n_ent, 48), rng.integers(0, n_rel, 48), rng.integers(0, n_ent, 48)]
    m = KEModel(_args(lr=lr, neg_adversarial_sampling=True, regularization_coef=reg), model, n_ent, n_rel, 400, 19.9)
    hp = ko.Hyper(model=model, hidden_dim=400, gamma=19.9, lr=lr, reg_coef=reg, adversarial=True)
    o = list(ko.init_tables(hp, n_ent, n_rel, seed=9))
    m.entity_emb.emb.copy_(o[0])
    m.relation_emb.emb.copy_(o[2])
    o = [x.double() for x in o]     # the oracle's own fp32 rounding moves a few updated rows by ~1e-5 over 6 steps
    sampler = DeviceGraphSampler(*tr, n_ent, B, N, seed=5) if device_sampler else TripleSampler(*tr, n_ent, n_rel, B, N, seed=5)
    try:
        logs = []
        for step in range(6):
            pos_g, neg_g = next(sampler)
            if device_sampler:
                b = pos_g.device_batch
                si = [x.cpu() for x in b.tensors()]
                neg_head = b.neg_head
            else:
                hl, tl = pos_g.all_edges()
                si = [pos_g.ndata["id"], hl, tl, pos_g.edata["id"], neg_g.ndata["id"]]
                neg_head = neg_g.neg_head
            m.forward(pos_g, neg_g, 0)
            m.update(0)
            ko.train_step(hp, *o, *si, B // N, N, N, neg_head)
            if step == 2:
                with th.no_grad():
                    for pg, ng in eval_batches(*va, n_ent, 16, False):
                        m.forward_test(pg, ng, logs, 0)
                assert len(logs) == 48
    finally:
        if device_sampler:
            sampler.s.close()
    th.cuda.synchronize()
    for got, want, what in ((m.entity_emb.emb, o[0], "entity table"), (m.entity_emb.state_sum, o[1], "entity state"),
                            (m.relation_emb.emb, o[2], "relation table"), (m.relation_emb.state_sum, o[3], "relation state")):
        w = want.numpy()
        np.testing.assert_allclose(got.cpu().numpy(), w, rtol=1e-4, atol=5e-6 * float(np.abs(w).max()), err_msg=what)


def test_update_after_an_evaluation_is_refused(fresh_handle):
    """forward_backward -> score_neg -> update: the evaluation has overwritten the step's gradients, so the update
    must be refused rather than apply them."""
    from dglke_b200 import _lib
    from dglke_b200.engine import StepEngine, DeviceTable, Hyper, score_neg
    from test_gpu_parity import _random_step
    hp = ko.Hyper(model="TransE_l2", hidden_dim=64, gamma=12.0, lr=0.1)
    ent, es, rel, rs = ko.init_tables(hp, 3000, 20, seed=8)
    dev = th.device("cuda", 0)
    e, e_s, r, r_s = (x.to(dev).contiguous() for x in (ent, es, rel, rs))
    ehp = Hyper(model="TransE_l2", hidden_dim=64, gamma=12.0, lr=0.1)
    eng = StepEngine(ehp, DeviceTable.from_tensors(e, e_s), DeviceTable.from_tensors(r, r_s), 0)
    si, C = _random_step(hp, 3000, 20, 256, 64, 64, False, seed=3)
    eng.forward_backward(*[si[k].to(dev) for k in ("node_ids", "head_local", "tail_local", "rel_ids", "neg_ids")],
                         64, 64, False)
    score_neg(ehp, e[:16], r[:16], e, 1, 16, 3000, False)
    before = e.clone()
    with pytest.raises(_lib.KgeError):
        eng.update()
    th.cuda.synchronize()
    assert th.equal(e, before)
