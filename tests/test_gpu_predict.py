"""Link prediction on the GPU: kge_topk alone against a host sort (exact, no tolerance), dglke_b200.predict against the
reference's ScoreInfer.topK fixtures (all six models x five exec modes, both score functions), an FB15k-shaped case
against torch.topk over the same device tiles, and the CLI on a checkpoint written by `python -m dglke_b200.train`."""
import glob
import os
import subprocess
import sys

import numpy as np
import pytest
import torch as th

from predict_f64 import brute_topk, cube64, list_keys
from test_gpu_eval_scores import allowed_error

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "predict")
U = 2.0 ** -24


@pytest.fixture(scope="module")
def handle():
    from dglke_b200 import _lib
    h = _lib.Handle(0)
    yield h
    h.close()


def run_topk(h, tiles, K, G):
    """Feeds tiles [(S [Q, N] float32, qgroup, qoff, cbase, cstride)] through kge_topk; returns the lists (numpy)."""
    from dglke_b200 import _lib
    dev = h.device
    ts = th.full((G, K), float("-inf"), device=dev)
    tk = th.full((G, K), -1, dtype=th.int64, device=dev)
    for S, qg, qo, cbase, cstride in tiles:
        S = th.as_tensor(S).to(dev).contiguous()
        qg = th.as_tensor(qg, dtype=th.int64).to(dev)
        qo = th.as_tensor(qo, dtype=th.int64).to(dev)
        Q, N = S.shape
        _lib.check(h.lib.kge_topk(h.raw, S.data_ptr(), N, Q, N, qg.data_ptr(), qo.data_ptr(), cbase, cstride, K, G,
                                  ts.data_ptr(), tk.data_ptr(), h.stream()))
    th.cuda.synchronize()
    return ts.cpu().numpy(), tk.cpu().numpy()


def host_topk(tiles, K, G):
    sc, gr, ky = [], [], []
    for S, qg, qo, cbase, cstride in tiles:
        S = np.asarray(S, np.float32)
        Q, N = S.shape
        sc.append(S.ravel())
        gr.append(np.repeat(np.asarray(qg), N))
        ky.append((np.asarray(qo)[:, None] + (cbase + np.arange(N))[None, :] * cstride).ravel())
    return brute_topk(np.concatenate(sc), np.concatenate(gr), np.concatenate(ky), G, K)


def assert_same(got, want):
    np.testing.assert_array_equal(got[1], want[1])
    np.testing.assert_array_equal(got[0].view(np.uint32), want[0].view(np.uint32))


def column_tiles(rng, Q, N, n_tiles, groups, fill=None):
    """n_tiles tiles over consecutive column blocks of the same Q rows; row q belongs to groups[q]."""
    qoff = np.arange(Q, dtype=np.int64) * (N * n_tiles)
    out = []
    for t in range(n_tiles):
        S = rng.standard_normal((Q, N)).astype(np.float32) if fill is None else np.full((Q, N), fill, np.float32)
        out.append((S, groups, qoff, t * N, 1))
    return out


# ---------------------------------------------------------------------------------------------------- kge_topk alone
@pytest.mark.parametrize("K", [1, 10, 1000, 1024])
def test_topk_matches_host_sort(handle, K):
    rng = np.random.default_rng(K)
    Q, N = 37, 5000                                  # N is not a multiple of the 4 096-column segment
    groups = np.repeat(np.arange(5), [3, 9, 1, 20, 4])
    tiles = column_tiles(rng, Q, N, 3, groups)
    got = run_topk(handle, tiles, K, 5)
    assert_same(got, host_topk(tiles, K, 5))
    assert_same(run_topk(handle, tiles, K, 5), got)              # a second run gives the same bits


def test_topk_ten_thousand_small_groups(handle):
    rng = np.random.default_rng(1)
    Q, N = 10000, 300
    tiles = column_tiles(rng, Q, N, 2, np.arange(Q))
    assert_same(run_topk(handle, tiles, 10, Q), host_topk(tiles, 10, Q))


def test_topk_one_group_many_tiles(handle):
    rng = np.random.default_rng(2)
    tiles = [(rng.standard_normal((8, 3000)).astype(np.float32), np.zeros(8, np.int64),
              np.arange(8, dtype=np.int64) * 100000 + t * 800000, 0, 1) for t in range(20)]
    assert_same(run_topk(handle, tiles, 100, 1), host_topk(tiles, 100, 1))


@pytest.mark.parametrize("K", [7, 1000, 1024])
def test_topk_all_equal_tiles(handle, K):
    """Every element ties: more survivors than K in every segment, the keys decide (the radix-select path)."""
    rng = np.random.default_rng(3)
    one = column_tiles(rng, 4, 9000, 1, np.zeros(4, np.int64), fill=1.5)
    assert_same(run_topk(handle, one, K, 1), host_topk(one, K, 1))
    stream = column_tiles(rng, 3, 5000, 5, np.array([0, 0, 1]), fill=-2.0)
    assert_same(run_topk(handle, stream, K, 2), host_topk(stream, K, 2))


def test_topk_nan_inf_and_signed_zeros(handle):
    rng = np.random.default_rng(4)
    Q, N = 6, 7000
    tiles = []
    for t in range(3):
        S = rng.standard_normal((Q, N)).astype(np.float32)
        u = rng.random((Q, N))
        S[u < 0.1] = np.nan
        S[(u >= 0.1) & (u < 0.15)] = np.inf
        S[(u >= 0.15) & (u < 0.2)] = -np.inf
        S[(u >= 0.2) & (u < 0.25)] = 0.0
        S[(u >= 0.25) & (u < 0.3)] = -0.0
        tiles.append((S, np.array([0, 0, 1, 1, 1, 2]), np.arange(Q, dtype=np.int64) * 3 * N, t * N, 1))
    for K in (50, 1024):
        assert_same(run_topk(handle, tiles, K, 3), host_topk(tiles, K, 3))
    # a list that only ever sees -inf and NaN: the -inf elements enter, the NaNs do not
    S = np.full((2, 300), -np.inf, np.float32)
    S[:, ::3] = np.nan
    t = [(S, np.zeros(2, np.int64), np.array([0, 300]), 0, 1)]
    got = run_topk(handle, t, 1000, 1)
    assert_same(got, host_topk(t, 1000, 1))
    assert (got[1][0] >= 0).sum() == 400 and (got[1][0, 400:] == -1).all()


def test_topk_fewer_elements_than_k(handle):
    rng = np.random.default_rng(5)
    tiles = column_tiles(rng, 2, 100, 1, np.array([0, 1]))
    got = run_topk(handle, tiles, 1000, 3)
    assert_same(got, host_topk(tiles, 1000, 3))
    assert (got[1][2] == -1).all() and np.isneginf(got[0][2]).all()    # list 2 saw nothing


def test_topk_strided_keys(handle):
    """batch_tail's layout: column stride |R| |T|, rows of many lists in one tile."""
    rng = np.random.default_rng(6)
    nR, nT, nH = 3, 40, 5000
    q = np.arange(nR * nT)
    k, j = q // nR, q % nR
    S = rng.standard_normal((len(q), nH)).astype(np.float32)
    tiles = [(S[:, :2500], k, j * nT + k, 0, nR * nT), (S[:, 2500:], k, j * nT + k, 2500, nR * nT)]
    assert_same(run_topk(handle, tiles, 20, nT), host_topk(tiles, 20, nT))


def test_topk_refuses_k_above_the_limit(handle):
    from dglke_b200 import _lib
    with pytest.raises(_lib.KgeError, match="KGE_TOPK_MAX=1024"):
        run_topk(handle, column_tiles(np.random.default_rng(0), 2, 10, 1, np.zeros(2, np.int64)), 1025, 1)


# ------------------------------------------------------------------------------------------- end to end, golden files
GOLDEN_FILES = sorted(glob.glob(os.path.join(GOLDEN, "predict_*.npz")))


def _bound(model, D, gamma, s64, sc):
    return allowed_error(model, D, gamma, th.from_numpy(np.asarray(s64, np.float64)),
                         th.from_numpy(np.asarray(sc, np.float64))).numpy()


@pytest.mark.parametrize("path", GOLDEN_FILES, ids=lambda p: os.path.basename(p)[8:-4])
def test_predict_matches_reference_fixture(path):
    from dglke_b200.predict import Predictor, infer_hyper, Plan
    z = np.load(path)
    model, mode, K, sfunc = str(z["model"]), str(z["exec_mode"]), int(z["k"]), str(z["score_func"])
    cfg = dict(model_name=model, hidden_dim=int(z["hidden_dim"]), gamma=float(z["gamma"]), double_ent=bool(z["double_ent"]),
               double_rel=bool(z["double_rel"]), dataset="g")
    hp = infer_hyper(cfg, sfunc)
    ent, rel = z["ent"], z["rel"]
    H, R, T = (z[n] if n in z else None for n in ("list_h", "list_r", "list_t"))
    p = Predictor(hp, ent, rel, 0)
    try:
        res = p.topk(H, R, T, mode, K, sfunc)
    finally:
        p.close()
    Hn = H if H is not None else np.arange(len(ent))
    Rn = R if R is not None else np.arange(len(rel))
    Tn = T if T is not None else np.arange(len(ent))
    s64, sc = cube64(model, ent, rel, Hn, Rn, Tn, hp.gamma, hp.hidden_dim, mode == "triplet_wise")
    tol = _bound(model, hp.entity_dim, hp.gamma, s64, sc)
    plan = Plan(mode, len(Hn), len(Rn), len(Tn))
    g, keys = list_keys(mode, len(Hn), len(Rn), len(Tn))
    want_k = brute_topk(s64.ravel(), g, keys, plan.n_lists, K + 1)[1]    # one more: the gap below the last entry
    lens = z["lens"]
    assert [len(x[3]) for x in res] == lens.tolist()
    off = np.concatenate([[0], np.cumsum(lens)])
    flat_s, flat_t = s64.ravel(), tol.ravel()
    f = (lambda x: -np.logaddexp(0.0, -x)) if sfunc == "logsigmoid" else (lambda x: x)
    for gi, (h, r, t, s) in enumerate(res):
        gh, gr, gt = (z[c][off[gi]:off[gi + 1]] for c in ("res_h", "res_r", "res_t"))
        wk = want_k[gi][want_k[gi] >= 0]
        ws, wt = flat_s[wk], flat_t[wk]
        i, j, k = plan.decode(_keys_of(plan, Hn, Rn, Tn, h, r, t, wk))
        mine, mtol = flat_s[_flat(plan, i, j, k)], flat_t[_flat(plan, i, j, k)]
        for pos in range(lens[gi]):
            # a position whose float64 neighbours are further apart than both bounds holds one triple only
            near = [q for q in (pos - 1, pos + 1) if 0 <= q < len(ws)]
            if all(abs(ws[pos] - ws[q]) > 2 * (wt[pos] + wt[q]) for q in near):
                assert (h[pos], r[pos], t[pos]) == (gh[pos], gr[pos], gt[pos]), (path, gi, pos)
            else:
                assert abs(mine[pos] - ws[pos]) <= mtol[pos] + wt[pos], (path, gi, pos)
        err = np.abs(s.astype(np.float64) - f(mine))
        assert (err <= mtol + 8 * U * np.abs(f(mine))).all(), (path, gi, err, mtol)


def _keys_of(plan, Hn, Rn, Tn, h, r, t, wk):
    """The keys of the returned triples: the expected key where the triple matches it, else the first key of the triple
    (the lists may repeat ids; a repeated triple has the same score)."""
    i, j, k = plan.decode(wk)
    out = []
    for n in range(len(h)):
        if n < len(wk) and (Hn[i[n]], Rn[j[n]], Tn[k[n]]) == (h[n], r[n], t[n]):
            out.append(wk[n])
            continue
        if plan.mode == "triplet_wise":
            c = np.nonzero((Hn == h[n]) & (Rn == r[n]) & (Tn == t[n]))[0]
            out.append(c[0])
        else:
            ii, jj, kk = np.nonzero(Hn == h[n])[0][0], np.nonzero(Rn == r[n])[0][0], np.nonzero(Tn == t[n])[0][0]
            out.append((ii * plan.nR + jj) * plan.nT + kk)
    return np.asarray(out, np.int64)


def _flat(plan, i, j, k):
    return i if plan.mode == "triplet_wise" else (i * plan.nR + j) * plan.nT + k


def test_rotate_none_reproduces_the_phase_quirk():
    """Under --score_func none InferModel's RotatE phase scale is 2 / hidden_dim: the fixture agrees with that and not
    with the trained scale (gamma + 2) / hidden_dim."""
    z = np.load(os.path.join(GOLDEN, "predict_RotatE_all_none.npz"))
    ent, rel, hid, gamma = z["ent"], z["rel"], int(z["hidden_dim"]), float(z["gamma"])
    H, R = z["list_h"], z["list_r"]
    T = np.arange(len(ent))
    s0, _ = cube64("RotatE", ent, rel, H, R, T, 0.0, hid)
    sg, _ = cube64("RotatE", ent, rel, H, R, T, gamma, hid)
    g, keys = list_keys("all", len(H), len(R), len(T))
    k0 = brute_topk(s0.ravel(), g, keys, 1, 10)[1][0]
    kg = brute_topk((sg - gamma).ravel(), g, keys, 1, 10)[1][0]
    assert not np.array_equal(k0, kg)
    i, j, k = k0 // (len(R) * len(T)), (k0 // len(T)) % len(R), k0 % len(T)
    np.testing.assert_array_equal(H[i], z["res_h"])
    np.testing.assert_array_equal(R[j], z["res_r"])
    np.testing.assert_array_equal(T[k], z["res_t"])


# ------------------------------------------------------------------------------------------------------------ at scale
def _torch_lists(p, plan, ids, K):
    """torch.topk over the same device tiles, ties resolved by a stable sort on the keys."""
    G = plan.n_lists
    run_s = [th.empty(0, device=p.device) for _ in range(G)]
    run_k = [th.empty(0, dtype=th.int64, device=p.device) for _ in range(G)]
    for S, qg, qo, cbase in p.tiles(plan, *ids):
        Q, N = S.shape
        keys = qo[:, None] + (cbase + th.arange(N, device=p.device))[None, :] * plan.cstride
        for g in th.unique(qg).tolist():
            m = qg == g
            s, k = th.cat([run_s[g], S[m].reshape(-1)]), th.cat([run_k[g], keys[m].reshape(-1)])
            kk = min(K, s.numel())
            thr = th.topk(s, kk).values[-1]
            sel = s >= thr
            s, k = s[sel], k[sel]
            o = th.argsort(k)
            s, k = s[o], k[o]
            o = th.sort(-s, stable=True).indices[:kk]
            run_s[g], run_k[g] = s[o], k[o]
    out_s = np.full((G, K), -np.inf, np.float32)
    out_k = np.full((G, K), -1, np.int64)
    for g in range(G):
        out_s[g, :run_s[g].numel()] = run_s[g].cpu().numpy()
        out_k[g, :run_k[g].numel()] = run_k[g].cpu().numpy()
    return out_s, out_k


@pytest.mark.parametrize("case", ["h_*_*_batch_head", "h_r_t_all_repeats"])
def test_predict_at_fb15k_scale_matches_torch_topk(case):
    from dglke_b200.engine import Hyper
    from dglke_b200.predict import Predictor, Plan
    rng = np.random.default_rng(7)
    n_ent, n_rel, D = 14951, 1345, 400
    hp = Hyper(model="TransE_l2", hidden_dim=D, gamma=0.0)
    ent = (rng.standard_normal((n_ent, D)) * 0.05).astype(np.float32)
    rel = (rng.standard_normal((n_rel, D)) * 0.05).astype(np.float32)
    p = Predictor(hp, ent, rel, 0)
    try:
        if case == "h_*_*_batch_head":
            H, R, T, mode, K = rng.integers(0, n_ent, 64), None, None, "batch_head", 10
        else:
            H, R, T, mode = rng.integers(0, n_ent, 16), rng.integers(0, n_rel, 50), rng.integers(0, 700, 3000), "all"
            K = 50
        nH = len(H)
        nR = n_rel if R is None else len(R)
        nT = n_ent if T is None else len(T)
        plan = Plan(mode, nH, nR, nT)
        ids = [None if x is None else th.from_numpy(np.asarray(x, np.int64)).to(p.device) for x in (H, R, T)]
        ts, tk = p.topk_keys(plan, *ids, K)
        want = _torch_lists(p, plan, ids, K)
    finally:
        p.close()
    assert_same((ts.cpu().numpy(), tk.cpu().numpy()), want)


# ------------------------------------------------------------------------------------------------------------------ CLI
def _env():
    env = dict(os.environ)
    env["PYTHONPATH"] = os.pathsep.join([os.path.join(ROOT, "dgl-ke_b200"), env.get("PYTHONPATH", "")])
    return env


@pytest.fixture(scope="module")
def checkpoint(tmp_path_factory):
    d = tmp_path_factory.mktemp("ckpt")
    fx = os.path.join(ROOT, "tests", "fixtures", "udd")
    r = subprocess.run([sys.executable, "-m", "dglke_b200.train", "--model_name", "TransE", "--dataset", "tiny",
                        "--format", "udd_hrt", "--data_path", fx, "--data_files", "entities.dict", "relations.dict",
                        "train.txt", "valid.txt", "test.txt", "--batch_size", "16", "--neg_sample_size", "4",
                        "--hidden_dim", "8", "--max_step", "20", "--log_interval", "10", "--save_path", str(d),
                        "--gpu", "0"], env=_env(), capture_output=True, text=True, cwd=str(d))
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
    (run,) = [os.path.join(d, x) for x in os.listdir(d) if x.startswith("TransE_tiny_")]
    assert os.path.exists(os.path.join(run, "tiny_TransE_l2_entity.npy"))
    return run, fx


CLI_CASES = [("h_r_t", "triplet_wise"), ("h_r_*", "all"), ("h_*_t", "batch_head"), ("*_r_t", "batch_rel"),
             ("h_*_*", "batch_head"), ("*_r_*", "batch_rel"), ("*_*_t", "batch_tail"), ("h_r_t", "batch_tail")]


@pytest.mark.parametrize("raw", [False, True])
@pytest.mark.parametrize("fmt,mode", CLI_CASES)
def test_cli_predict(checkpoint, tmp_path, fmt, mode, raw):
    from dglke_b200.predict import Predictor, infer_hyper, load_checkpoint, read_mapping, write_result
    run, fx = checkpoint
    e2i, i2e = read_mapping(os.path.join(fx, "entities.dict"))
    r2i, i2r = read_mapping(os.path.join(fx, "relations.dict"))
    lists = {"h": [3, 7, 3, 11], "r": [0, 2], "t": [5, 1, 9, 5]}
    if mode == "triplet_wise":
        lists = {"h": [3, 7, 3, 11], "r": [0, 2, 1, 1], "t": [5, 1, 9, 5]}
    files = []
    for side, c in zip("hrt", fmt.split("_")):
        if c == "*":
            continue
        path = str(tmp_path / ("%s.list" % side))
        names = [(i2r if side == "r" else i2e)[x] if raw else str(x) for x in lists[side]]
        with open(path, "w") as f:
            f.write("\n".join(names))                    # no newline after the last line
        files.append(path)
    from dglke_b200 import predict
    outs = []
    for n in range(2):
        out = str(tmp_path / ("out%d.tsv" % n))
        argv = ["--model_path", run, "--format", fmt, "--data_files", *files, "--exec_mode", mode, "--topK", "5",
                "--output", out, "--gpu", "0"]
        if raw:
            argv += ["--raw_data", "--entity_mfile", os.path.join(fx, "entities.dict"), "--rel_mfile",
                     os.path.join(fx, "relations.dict")]
        if fmt == "h_r_t" and mode == "triplet_wise":          # once through the module's command line
            r = subprocess.run([sys.executable, "-m", "dglke_b200.predict", *argv], env=_env(), capture_output=True,
                               text=True)
            assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
        else:
            predict.main(argv)
        outs.append(open(out, "rb").read())
    assert outs[0] == outs[1]
    # the same lists through the API
    config, ent, rel = load_checkpoint(run)
    p = Predictor(infer_hyper(config, "none"), ent, rel, 0)
    try:
        get = lambda s: np.asarray(lists[s]) if s in [x[0] for x in zip("hrt", fmt.split("_")) if x[1] != "*"] else None
        res = p.topk(get("h"), get("r"), get("t"), mode, 5)
    finally:
        p.close()
    want = str(tmp_path / "api.tsv")
    write_result(want, res, i2e if raw else None, i2r if raw else None)
    assert outs[0] == open(want, "rb").read()
    lines = outs[0].decode().split("\n")
    assert lines[0] == "head\trel\ttail\tscore" and lines[-1] == ""
    assert len(lines) - 2 == sum(len(x[3]) for x in res) > 0


def test_cli_refuses_cpu(checkpoint, tmp_path):
    run, _ = checkpoint
    r = subprocess.run([sys.executable, "-m", "dglke_b200.predict", "--model_path", run, "--format", "h_*_*",
                        "--data_files", "x"], env=_env(), capture_output=True, text=True)
    assert r.returncode != 0 and "needs --gpu" in r.stderr


def test_cli_matches_the_reference_output_file(tmp_path):
    """The reference's command line on DistMult tables (--format h_*_t --exec_mode batch_head --raw_data --topK 5, see
    tools/gen_predict_golden.py): the same lines, ids and names; the scores within their fp32 bounds.  The float64 gaps
    between neighbours in these lists are far above the bounds, so the order is not a near tie anywhere."""
    from dglke_b200 import predict
    z = np.load(os.path.join(GOLDEN, "cli_DistMult.npz"))
    ent, rel = z["ent"], z["rel"]
    np.save(str(tmp_path / "g_DistMult_entity.npy"), ent)
    np.save(str(tmp_path / "g_DistMult_relation.npy"), rel)
    with open(str(tmp_path / "config.json"), "w") as f:
        import json
        json.dump(dict(model_name="DistMult", hidden_dim=32, double_ent=False, double_rel=False, gamma=9.0,
                       dataset="g"), f)
    for name, n, c in (("entities.dict", len(ent), "e"), ("relations.dict", len(rel), "r")):
        (tmp_path / name).write_text("".join("%d\t%s%d\n" % (i, c, i) for i in range(n)))
    (tmp_path / "h.list").write_text("e3\ne17\ne41\n")
    (tmp_path / "t.list").write_text("e0\ne12\ne33\ne49\ne7\n")
    out = str(tmp_path / "out.tsv")
    predict.main(["--model_path", str(tmp_path), "--format", "h_*_t", "--data_files", str(tmp_path / "h.list"),
                  str(tmp_path / "t.list"), "--exec_mode", "batch_head", "--raw_data", "--entity_mfile",
                  str(tmp_path / "entities.dict"), "--rel_mfile", str(tmp_path / "relations.dict"), "--topK", "5",
                  "--output", out, "--gpu", "0"])
    got = open(out).read().split("\n")
    want = open(os.path.join(GOLDEN, "cli_DistMult.tsv")).read().split("\n")
    assert len(got) == len(want) and got[0] == want[0] == "head\trel\ttail\tscore" and got[-1] == want[-1] == ""
    rows = [(g.split("\t"), w.split("\t")) for g, w in zip(got[1:-1], want[1:-1])]
    assert all(g[:3] == w[:3] for g, w in rows)
    num = lambda x: int(x[1:])
    H, R, T = (np.array([num(w[c]) for _, w in rows]) for c in range(3))
    s64, sc = cube64("DistMult", ent, rel, H, R, T, 0.0, 32, triplet_wise=True)
    tol = _bound("DistMult", 32, 0.0, s64, sc)
    for lst in range(3):
        s = s64[5 * lst:5 * lst + 5]
        t = tol[5 * lst:5 * lst + 5]
        assert (np.diff(-s) > 2 * (t[1:] + t[:-1])).all()
    assert (np.abs(np.array([float(g[3]) for g, _ in rows]) - s64) <= tol).all()
