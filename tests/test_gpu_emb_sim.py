"""Embedding similarity on the GPU: kge_sim_tile and kge_sim_pairs against float64 within emb_sim_f64.sim64's per-function
bounds, self pairs and near-duplicates under l1 / l2, zero rows, dglke_b200.emb_sim against the reference's
EmbSimInfer.topK fixtures, an FB15k-shaped run against torch.topk over the same device tiles, and the CLI on a table
written by `python -m dglke_b200.train`."""
import glob
import os
import subprocess
import sys

import numpy as np
import pytest
import torch as th

from emb_sim_f64 import list_keys, sim64
from predict_f64 import brute_topk
from test_emb_sim_host import GOLDEN, fixture_lists

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FUNCS = ("cosine", "l2", "l1", "dot", "ext_jaccard")


@pytest.fixture(scope="module")
def handle():
    from dglke_b200 import _lib
    h = _lib.Handle(0)
    yield h
    h.close()


def sim_tile(h, func, L, R):
    from dglke_b200 import _lib
    L = th.as_tensor(L).to(h.device).contiguous()
    R = th.as_tensor(R).to(h.device).contiguous()
    out = th.empty((L.shape[0], R.shape[0]), device=h.device)
    _lib.check(h.lib.kge_sim_tile(h.raw, _lib.SIM_IDS[func], L.data_ptr(), L.shape[0], R.data_ptr(), R.shape[0],
                                  L.shape[1], out.data_ptr(), h.stream()))
    th.cuda.synchronize()
    return out.cpu().numpy()


def sim_pairs(h, func, L, R):
    from dglke_b200 import _lib
    L = th.as_tensor(L).to(h.device).contiguous()
    R = th.as_tensor(R).to(h.device).contiguous()
    out = th.empty(L.shape[0], device=h.device)
    _lib.check(h.lib.kge_sim_pairs(h.raw, _lib.SIM_IDS[func], L.data_ptr(), R.data_ptr(), L.shape[0], L.shape[1],
                                   out.data_ptr(), h.stream()))
    th.cuda.synchronize()
    return out.cpu().numpy()


def assert_within(got, s64, bound, what):
    err = np.abs(got.astype(np.float64) - s64)
    assert np.isfinite(got).all(), what
    assert (err <= bound).all(), (what, float((err / bound).max()))


# ------------------------------------------------------------------------------------------------ kernels vs float64
@pytest.mark.parametrize("dim", [1, 7, 32, 33, 400, 401, 800])
@pytest.mark.parametrize("func", FUNCS)
def test_sim_tile_and_pairs_against_float64(handle, func, dim):
    """nL = 150 and nR = 300 are multiples of neither tile (128 x 256 GEMM, 64 x 64 difference tiles)."""
    rng = np.random.default_rng(dim * 10 + FUNCS.index(func))
    L = (rng.standard_normal((150, dim)) * 0.3).astype(np.float32)
    R = (rng.standard_normal((300, dim)) * 0.3).astype(np.float32)
    R[:40] = L[:40] + (rng.standard_normal((40, dim)) * 0.01).astype(np.float32)     # close pairs: |s| near its max
    s64, bound = sim64(func, L, R)
    assert_within(sim_tile(handle, func, L, R), s64, bound, (func, dim, "tile"))
    p64, pbound = sim64(func, L, R[:150], pairwise=True)
    assert_within(sim_pairs(handle, func, L, R[:150]), p64, pbound, (func, dim, "pairs"))


@pytest.mark.parametrize("func", FUNCS)
def test_sim_tile_wide_rows(handle, func):
    rng = np.random.default_rng(11)
    L = (rng.standard_normal((5, 10000)) * 0.05).astype(np.float32)
    R = (rng.standard_normal((9, 10000)) * 0.05).astype(np.float32)
    R[0] = L[0]
    s64, bound = sim64(func, L, R)
    assert_within(sim_tile(handle, func, L, R), s64, bound, (func, "wide"))
    p64, pbound = sim64(func, L, R[:5], pairwise=True)
    assert_within(sim_pairs(handle, func, L, R[:5]), p64, pbound, (func, "wide pairs"))


# ------------------------------------------------------------------------------------- self pairs and near duplicates
@pytest.mark.parametrize("func", ["l1", "l2"])
def test_self_pairs_are_negative_zero_and_near_duplicates_rank_in_float64_order(handle, func):
    """Every row against itself scores exactly -0.0 (sign bit set), in the tile and in the pairs.  Rows x + delta_m,
    |delta_m| ~ 1e-5 |x| (m + 1) in random directions, rank in float64 order: the expanded form |x|^2 + |y|^2 - 2 x.y
    has an error of about sqrt(u) |x| here, far above the gaps, and fails this."""
    rng = np.random.default_rng(3)
    D = 400
    X = (rng.standard_normal((70, D)) * 0.3).astype(np.float32)
    S = sim_tile(handle, func, X, X)
    diag = np.diagonal(S)
    assert (diag == 0).all() and np.signbit(diag).all()
    P = sim_pairs(handle, func, X, X)
    assert (P == 0).all() and np.signbit(P).all()
    x = X[0].astype(np.float64)
    nx = np.linalg.norm(x)
    dirs = rng.standard_normal((60, D))
    dirs /= np.linalg.norm(dirs, axis=1, keepdims=True)
    Y = (x[None, :] + 1e-5 * nx * (np.arange(60)[:, None] + 1) * dirs).astype(np.float32)
    Y = Y[rng.permutation(60)]
    s64, _ = sim64(func, X[:1], Y)
    got = sim_tile(handle, func, X[:1], Y)[0]
    np.testing.assert_array_equal(np.argsort(-got, kind="stable"), np.argsort(-s64[0], kind="stable"))


def test_l2_query_finds_itself_first():
    from dglke_b200.emb_sim import EmbSim
    rng = np.random.default_rng(4)
    emb = (rng.standard_normal((3000, 64)) * 0.3).astype(np.float32)
    s = EmbSim(emb, 0)
    try:
        q = np.array([5, 2999, 17, 5])
        for func in ("l1", "l2"):
            res = s.topk(q, None, "batch_left", 5, func)
            for i, (l, r, sc) in enumerate(res):
                assert (l == q[i]).all() and r[0] == q[i] and sc[0] == 0 and np.signbit(sc[0])
    finally:
        s.close()


# ----------------------------------------------------------------------------------------------------------- zero rows
@pytest.mark.parametrize("mode", ["all", "batch_left", "pairwise"])
def test_zero_rows_never_enter_a_list_as_nan(mode):
    """cosine of a zero row and ext_jaccard of two zero rows are NaN (as in the reference); no list holds them."""
    from dglke_b200.emb_sim import EmbSim
    rng = np.random.default_rng(5)
    emb = (rng.standard_normal((300, 33)) * 0.3).astype(np.float32)
    zeros = [0, 7, 150]
    emb[zeros] = 0
    s = EmbSim(emb, 0)
    try:
        for func in ("cosine", "ext_jaccard"):
            res = s.topk(None, None, mode, 20, func)
            for l, r, sc in res:
                assert not np.isnan(sc).any()
                if func == "cosine":
                    assert not np.isin(l, zeros).any() and not np.isin(r, zeros).any()
                else:
                    assert not (np.isin(l, zeros) & np.isin(r, zeros)).any()
            if mode == "batch_left":
                assert all(len(res[z][0]) == (0 if func == "cosine" else 20) for z in zeros)
    finally:
        s.close()


# ------------------------------------------------------------------------------------------- end to end, golden files
GOLDEN_FILES = sorted(glob.glob(os.path.join(GOLDEN, "sim_*.npz")))


@pytest.mark.parametrize("path", GOLDEN_FILES, ids=lambda p: os.path.basename(p)[4:-4])
def test_emb_sim_matches_reference_fixture(path):
    """The same (left, right) lists as the reference wherever the float64 neighbours of a position are further apart
    than their bounds; elsewhere (near ties, exact ties such as self pairs under l1 / l2 or (i, j) against (j, i)) the
    scores agree within the bounds.  Every score is within its bound of float64."""
    from dglke_b200.emb_sim import EmbSim, Plan
    z = np.load(path)
    mode, K, sim = str(z["exec_mode"]), int(z["k"]), str(z["sim_func"])
    emb, left, right, Ln, Rn = fixture_lists(z)
    s = EmbSim(emb, 0)
    try:
        res = s.topk(left, right, mode, K, sim)
    finally:
        s.close()
    s64, bound = sim64(sim, emb[Ln], emb[Rn], pairwise=mode == "pairwise")
    plan = Plan(mode, len(Ln), len(Rn))
    g, keys = list_keys(mode, len(Ln), len(Rn))
    ws, wk = brute_topk(s64.ravel(), g, keys, plan.n_lists, K + 1)      # one more: the gap below the last entry
    score_of, bound_of = {}, {}
    i, j = plan.decode(keys)
    for a, b, sc, bd in zip(Ln[i].tolist(), Rn[j].tolist(), s64.ravel().tolist(), bound.ravel().tolist()):
        score_of[(a, b)], bound_of[(a, b)] = sc, bd
    lens = z["lens"]
    assert [len(x[2]) for x in res] == lens.tolist()
    off = np.concatenate([[0], np.cumsum(lens)])
    for gi, (l, r, sc) in enumerate(res):
        gl, gr = z["res_l"][off[gi]:off[gi + 1]], z["res_r"][off[gi]:off[gi + 1]]
        m = wk[gi] >= 0
        w = ws[gi][m]
        wb = np.array([bound_of[p] for p in zip(Ln[plan.decode(wk[gi][m])[0]].tolist(),
                                                Rn[plan.decode(wk[gi][m])[1]].tolist())])
        for pos in range(lens[gi]):
            near = [q for q in (pos - 1, pos + 1) if 0 <= q < len(w)]
            if all(abs(w[pos] - w[q]) > 2 * (wb[pos] + wb[q]) for q in near):
                assert (l[pos], r[pos]) == (gl[pos], gr[pos]), (path, gi, pos)
            else:
                assert abs(score_of[(l[pos], r[pos])] - w[pos]) <= bound_of[(l[pos], r[pos])] + wb[pos], (path, gi, pos)
        mine = np.array([score_of[p] for p in zip(l.tolist(), r.tolist())])
        mb = np.array([bound_of[p] for p in zip(l.tolist(), r.tolist())])
        assert (np.abs(sc.astype(np.float64) - mine) <= mb).all(), (path, gi)
        if sim in ("l1", "l2"):
            selfp = l == r
            assert (sc[selfp] == 0).all() and np.signbit(sc[selfp]).all()


# ------------------------------------------------------------------------------------------------------------ at scale
def _torch_lists(s, plan, func, K):
    """torch over the same device tiles: per row, the running list and the tile's row sorted by (score descending, key
    ascending) with two stable sorts, the first K kept."""
    out_s = np.full((plan.n_lists, K), -np.inf, np.float32)
    out_k = np.full((plan.n_lists, K), -1, np.int64)
    run = {}
    for S, (b, e), qg, qo, cbase in s.tiles(plan, func, None, None, K):
        Q, N = S.shape
        keys = qo[:, None] + cbase + th.arange(N, device=S.device)[None, :]
        rs, rk = run.get((b, e), (th.empty((Q, 0), device=S.device), th.empty((Q, 0), dtype=th.int64, device=S.device)))
        vs, vk = th.cat([rs, S], 1), th.cat([rk, keys], 1)
        o = th.argsort(vk, dim=1, stable=True)
        vs, vk = th.gather(vs, 1, o), th.gather(vk, 1, o)
        o = th.sort(-vs, dim=1, stable=True).indices[:, :K]
        run[(b, e)] = (th.gather(vs, 1, o), th.gather(vk, 1, o))
    for (b, e), (rs, rk) in run.items():
        out_s[b:e], out_k[b:e] = rs.cpu().numpy(), rk.cpu().numpy()
    return out_s, out_k


@pytest.mark.parametrize("func", ["dot", "l2"])
def test_fb15k_shaped_batch_left_matches_torch(func):
    from dglke_b200.emb_sim import EmbSim, Plan
    rng = np.random.default_rng(8)
    emb = (rng.standard_normal((14951, 400)) * 0.05).astype(np.float32)
    s = EmbSim(emb, 0)
    try:
        plan = Plan("batch_left", 14951, 14951)
        got = s.topk_keys(plan, func, None, None, 10)
        want = _torch_lists(s, plan, func, 10)
    finally:
        s.close()
    np.testing.assert_array_equal(got[1], want[1])
    np.testing.assert_array_equal(got[0].view(np.uint32), want[0].view(np.uint32))


# ------------------------------------------------------------------------------------------------------------------ CLI
def _env():
    env = dict(os.environ)
    env["PYTHONPATH"] = os.pathsep.join([os.path.join(ROOT, "dgl-ke_b200"), env.get("PYTHONPATH", "")])
    return env


@pytest.fixture(scope="module")
def trained_table(tmp_path_factory):
    d = tmp_path_factory.mktemp("ckpt")
    fx = os.path.join(ROOT, "tests", "fixtures", "udd")
    r = subprocess.run([sys.executable, "-m", "dglke_b200.train", "--model_name", "TransE", "--dataset", "tiny",
                        "--format", "udd_hrt", "--data_path", fx, "--data_files", "entities.dict", "relations.dict",
                        "train.txt", "valid.txt", "test.txt", "--batch_size", "16", "--neg_sample_size", "4",
                        "--hidden_dim", "8", "--max_step", "20", "--log_interval", "10", "--save_path", str(d),
                        "--gpu", "0"], env=_env(), capture_output=True, text=True, cwd=str(d))
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
    (run,) = [os.path.join(d, x) for x in os.listdir(d) if x.startswith("TransE_tiny_")]
    path = os.path.join(run, "tiny_TransE_l2_entity.npy")
    assert os.path.exists(path)
    return path, os.path.join(fx, "entities.dict")


CLI_CASES = [("l_r", "pairwise"), ("*", "pairwise"), ("l_r", "all"), ("l_*", "all"), ("*_r", "all"), ("*", "all"),
             ("l_r", "batch_left"), ("l_*", "batch_left"), ("*_r", "batch_left"), ("*", "batch_left")]


@pytest.mark.parametrize("raw", [False, True])
@pytest.mark.parametrize("fmt,mode", CLI_CASES)
def test_cli_emb_sim(trained_table, tmp_path, fmt, mode, raw):
    from dglke_b200 import emb_sim
    from dglke_b200.predict import read_mapping
    emb_file, mfile = trained_table
    _, i2e = read_mapping(mfile)
    lists = {"l": [3, 7, 3, 11], "r": [5, 1, 9, 5] if mode == "pairwise" else [5, 1, 9, 5, 20]}
    files, given = [], {"l": fmt[0] != "*", "r": fmt[-1] != "*"}
    for side in "lr":
        if not given[side]:
            continue
        path = str(tmp_path / ("%s.list" % side))
        with open(path, "w") as f:
            f.write("\n".join(i2e[x] if raw else str(x) for x in lists[side]))      # no newline after the last line
        files.append(path)
    outs = []
    for n in range(2):
        out = str(tmp_path / ("out%d.tsv" % n))
        argv = ["--emb_file", emb_file, "--format", fmt, "--exec_mode", mode, "--topK", "6", "--sim_func", "l2",
                "--output", out, "--gpu", "0"] + (["--data_files"] + files if files else [])
        if raw:
            argv += ["--raw_data", "--mfile", mfile]
        if fmt == "l_r" and mode == "pairwise":          # once through the module's command line
            r = subprocess.run([sys.executable, "-m", "dglke_b200.emb_sim", *argv], env=_env(), capture_output=True,
                               text=True)
            assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
        else:
            emb_sim.main(argv)
        outs.append(open(out, "rb").read())
    assert outs[0] == outs[1]
    s = emb_sim.EmbSim(emb_sim.load_table(emb_file), 0)
    try:
        res = s.topk(np.asarray(lists["l"]) if given["l"] else None, np.asarray(lists["r"]) if given["r"] else None,
                     mode, 6, "l2")
    finally:
        s.close()
    want = str(tmp_path / "api.tsv")
    emb_sim.write_result(want, res, i2e if raw else None)
    assert outs[0] == open(want, "rb").read()
    lines = outs[0].decode().split("\n")
    assert lines[0] == "left\tright\tscore" and lines[-1] == ""
    assert len(lines) - 2 == sum(len(x[2]) for x in res) > 0


def test_cli_refuses_cpu(trained_table):
    emb_file, _ = trained_table
    r = subprocess.run([sys.executable, "-m", "dglke_b200.emb_sim", "--emb_file", emb_file, "--format", "*"],
                       env=_env(), capture_output=True, text=True)
    assert r.returncode != 0 and "needs --gpu" in r.stderr


def test_cli_matches_the_reference_output_file(tmp_path):
    """The reference's command line (--format l_* --exec_mode batch_left --raw_data --sim_func l2 --topK 5, see
    tools/gen_emb_sim_golden.py): the same lines and names, each list led by the query itself at -0.0, the scores within
    their bounds of float64."""
    from dglke_b200 import emb_sim
    z = np.load(os.path.join(GOLDEN, "cli_l2.npz"))
    emb = z["emb"]
    np.save(str(tmp_path / "emb.npy"), emb)
    (tmp_path / "entities.dict").write_text("".join("%d\te%d\n" % (i, i) for i in range(len(emb))))
    (tmp_path / "l.list").write_text("e3\ne17\ne25\n")
    out = str(tmp_path / "out.tsv")
    emb_sim.main(["--mfile", str(tmp_path / "entities.dict"), "--emb_file", str(tmp_path / "emb.npy"), "--format", "l_*",
                  "--data_files", str(tmp_path / "l.list"), "--raw_data", "--exec_mode", "batch_left", "--topK", "5",
                  "--sim_func", "l2", "--output", out, "--gpu", "0"])
    got = open(out).read().split("\n")
    want = open(os.path.join(GOLDEN, "cli_l2.tsv")).read().split("\n")
    assert len(got) == len(want) and got[0] == want[0] == "left\tright\tscore" and got[-1] == want[-1] == ""
    rows = [(g.split("\t"), w.split("\t")) for g, w in zip(got[1:-1], want[1:-1])]
    assert all(g[:2] == w[:2] for g, w in rows)
    assert all(g[2] == "-0.0" for g, _ in rows[::5])
    num = lambda x: int(x[1:])
    L, R = (np.array([num(w[c]) for _, w in rows]) for c in range(2))
    s64, bound = sim64("l2", emb[L], emb[R], pairwise=True)
    assert (np.abs(np.array([float(g[2]) for g, _ in rows]) - s64) <= bound).all()
