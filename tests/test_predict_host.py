"""dglke_b200.predict without a GPU: the flag surface against the reference's infer_score.ArgParser (recorded), the list
and mapping readers, the tile plan of every format x exec mode against a brute force over the full cube, the TransE ->
TransE_l2 file lookup, the multi-GPU config.json writer, and the golden fixtures against a float64 restatement."""
import argparse
import glob
import json
import os
import zlib

import numpy as np
import pytest

from predict_f64 import brute_topk, cube64, list_keys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "predict")


def test_flags_match_the_reference_parser():
    from dglke_b200.predict import ArgParser
    want = json.load(open(os.path.join(GOLDEN, "predict_flags.json")))
    got = [dict(option=a.option_strings, dest=a.dest, type=getattr(a.type, "__name__", None), default=a.default,
                nargs=a.nargs, action=type(a).__name__) for a in ArgParser()._actions if a.dest != "help"]
    assert got == want


def test_readers_keep_a_last_line_without_newline(tmp_path):
    from dglke_b200.predict import read_id_list, read_mapping, read_name_list, read_lists
    (tmp_path / "ids").write_text("3\n14\n15")
    np.testing.assert_array_equal(read_id_list(str(tmp_path / "ids")), [3, 14, 15])
    (tmp_path / "map").write_text("0\talpha\n1\tbeta\n2\tgamma\n")
    n2i, i2n = read_mapping(str(tmp_path / "map"))
    assert n2i == {"alpha": 0, "beta": 1, "gamma": 2} and i2n == {0: "alpha", 1: "beta", 2: "gamma"}
    (tmp_path / "names").write_text("gamma\nalpha\ngamma")
    np.testing.assert_array_equal(read_name_list(str(tmp_path / "names"), n2i), [2, 0, 2])
    h, r, t, (i2e, i2r) = read_lists("h_*_t", [str(tmp_path / "names")] * 2, True, str(tmp_path / "map"),
                                     str(tmp_path / "map"))
    assert r is None and i2e == i2n and list(t) == [2, 0, 2]
    with pytest.raises(SystemExit):
        read_lists("h_r_t", [str(tmp_path / "ids")])


FORMATS = ("h_r_t", "h_r_*", "h_*_t", "*_r_t", "h_*_*", "*_r_*", "*_*_t")
MODES = ("triplet_wise", "all", "batch_head", "batch_rel", "batch_tail")


@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("mode", MODES)
def test_plan_against_the_full_cube(fmt, mode):
    """Tiles built from the plan (queries in batches of 5, candidates in blocks of 3) and a host merge give the brute
    force's lists, and every key decodes to its own (i, j, k)."""
    from dglke_b200.predict import Plan
    n_ent, n_rel = 9, 4
    rng = np.random.default_rng(zlib.crc32((fmt + mode).encode()))
    given = [c != "*" for c in fmt.split("_")]
    if mode == "triplet_wise":
        if not all(given):
            pytest.skip("triplet_wise takes three lists of one length")
        nH = nR = nT = 6
    else:
        nH, nR, nT = (l if g else a for l, g, a in zip((4, 3, 5), given, (n_ent, n_rel, n_ent)))
    plan = Plan(mode, nH, nR, nT)
    cube = rng.permutation(nH * (1 if mode == "triplet_wise" else nR * nT)).astype(np.float32)
    K = 4
    g_all, k_all = list_keys(mode, nH, nR, nT)
    want = brute_topk(cube, g_all, k_all, plan.n_lists, K)
    # the plan's tiles
    sc, gr, ky = [], [], []
    if mode == "triplet_wise":
        for b in range(0, nH, 4):
            n = min(4, nH - b)
            sc.append(cube[b:b + n]); gr.append(np.zeros(n, np.int64)); ky.append(b + np.arange(n))
    else:
        c3 = cube.reshape(nH, nR, nT)
        for qb in range(0, plan.n_queries, 5):
            qe = min(plan.n_queries, qb + 5)
            (a, b), g, off = plan.queries(qb, qe)
            assert (np.diff(g) != 0).sum() == len(np.unique(g)) - 1          # a list's rows are consecutive
            for c0 in range(0, plan.n_cand, 3):
                c = np.arange(c0, min(plan.n_cand, c0 + 3))
                S = c3[c[None, :], a[:, None], b[:, None]] if plan.head_candidates else c3[a[:, None], b[:, None], c[None, :]]
                keys = off[:, None] + c[None, :] * plan.cstride
                i, j, k = plan.decode(keys)
                np.testing.assert_array_equal(c3[i, j, k], S)
                sc.append(S.ravel()); gr.append(np.repeat(g, len(c))); ky.append(keys.ravel())
    got = brute_topk(np.concatenate(sc), np.concatenate(gr), np.concatenate(ky), plan.n_lists, K)
    np.testing.assert_array_equal(got[1], want[1])
    np.testing.assert_array_equal(got[0], want[0])
    assert plan.n_lists == {"triplet_wise": 1, "all": 1, "batch_head": nH, "batch_rel": nR, "batch_tail": nT}[mode]


def test_transe_checkpoint_found_under_transe_l2(tmp_path):
    from dglke_b200.predict import checkpoint_files, load_checkpoint
    for side in ("entity", "relation"):
        np.save(str(tmp_path / ("ds_TransE_l2_%s.npy" % side)), np.zeros((3, 4), np.float32))
    json.dump(dict(model_name="TransE", dataset="ds", hidden_dim=4, gamma=1.0, double_ent=False, double_rel=False),
              open(str(tmp_path / "config.json"), "w"))
    e, r = checkpoint_files(str(tmp_path), "ds", "TransE")
    assert e.endswith("ds_TransE_l2_entity.npy") and r.endswith("ds_TransE_l2_relation.npy")
    cfg, ent, rel = load_checkpoint(str(tmp_path))
    assert ent.shape == (3, 4) and cfg["model_name"] == "TransE"
    with pytest.raises(SystemExit):
        checkpoint_files(str(tmp_path), "ds", "DistMult")


def test_refusals(tmp_path):
    from dglke_b200 import predict
    json.dump(dict(model_name="TransR", dataset="ds"), open(str(tmp_path / "config.json"), "w"))
    with pytest.raises(SystemExit, match="TransR"):
        predict.load_checkpoint(str(tmp_path))
    with pytest.raises(SystemExit, match="needs --gpu"):
        predict.main(["--model_path", str(tmp_path), "--format", "h_*_*", "--data_files", "x"])


def test_infer_hyper_gamma_and_rotate_phase_scale():
    from dglke_b200.predict import infer_hyper
    cfg = dict(model_name="RotatE", hidden_dim=40, gamma=9.0, double_ent=True, double_rel=False)
    assert infer_hyper(cfg, "none").gamma == 0.0 and infer_hyper(cfg, "none").emb_init == 2.0 / 40
    assert infer_hyper(cfg, "logsigmoid").emb_init == 11.0 / 40
    assert infer_hyper(dict(cfg, model_name="TransE"), "none").model == "TransE_l2"


def test_multi_gpu_config_writer(tmp_path):
    """_multi_gpu_worker's rank 0 writes config.json through save_config, as save_model does."""
    import inspect
    from dglke_b200 import train, utils
    args = argparse.Namespace(model_name="DistMult", dataset="ds", hidden_dim=8, gamma=12.0, double_ent=False,
                              double_rel=False, save_path=str(tmp_path), gpu=[0, 1])
    utils.save_config(args)
    cfg = json.load(open(str(tmp_path / "config.json")))
    assert cfg["model_name"] == "DistMult" and cfg["gpu"] == [0, 1] and cfg["emp_file"] is None
    assert "save_config(args)" in inspect.getsource(train._multi_gpu_worker)


GOLDEN_FILES = sorted(glob.glob(os.path.join(GOLDEN, "predict_*.npz")))


@pytest.mark.parametrize("path", GOLDEN_FILES, ids=lambda p: os.path.basename(p)[8:-4])
def test_fixture_against_float64(path):
    """The reference's lists are the float64 brute force's (up to exact ties, which its argsort breaks arbitrarily),
    and its scores are the float64 scores to fp32 accuracy."""
    from dglke_b200.predict import Plan
    z = np.load(path)
    model, mode, K, sfunc = str(z["model"]), str(z["exec_mode"]), int(z["k"]), str(z["score_func"])
    gamma = float(z["gamma"]) if sfunc == "logsigmoid" else 0.0
    ent, rel = z["ent"], z["rel"]
    H, R, T = (z[n] if n in z else None for n in ("list_h", "list_r", "list_t"))
    Hn = H if H is not None else np.arange(len(ent))
    Rn = R if R is not None else np.arange(len(rel))
    Tn = T if T is not None else np.arange(len(ent))
    s64, _ = cube64(model, ent, rel, Hn, Rn, Tn, gamma, int(z["hidden_dim"]), mode == "triplet_wise")
    plan = Plan(mode, len(Hn), len(Rn), len(Tn))
    g, keys = list_keys(mode, len(Hn), len(Rn), len(Tn))
    ws, wk = brute_topk(s64.ravel(), g, keys, plan.n_lists, K)
    off = np.concatenate([[0], np.cumsum(z["lens"])])
    # float64 score of every (head, rel, tail) of the cube (a repeated id in a list gives the same triple and score)
    i, j, k = plan.decode(keys)
    score_of = dict(zip(zip(Hn[i].tolist(), Rn[j].tolist(), Tn[k].tolist()), s64.ravel().tolist()))
    for gi in range(plan.n_lists):
        m = wk[gi] >= 0
        i, j, k = plan.decode(wk[gi][m])
        sl = slice(off[gi], off[gi + 1])
        got = list(zip(z["res_h"][sl].tolist(), z["res_r"][sl].tolist(), z["res_t"][sl].tolist()))
        want = list(zip(Hn[i].tolist(), Rn[j].tolist(), Tn[k].tolist()))
        s = ws[gi][m]
        assert len(got) == len(want)
        for pos in range(len(want)):
            # exact float64 ties (TransE with h = t scores -|r| for every such entity) are broken arbitrarily by the
            # reference's argsort: there only the score has to agree
            tie = np.isclose(s, s[pos], rtol=1e-9, atol=1e-12).sum() > 1
            assert got[pos] == want[pos] or (tie and np.isclose(score_of[got[pos]], s[pos], rtol=1e-9, atol=1e-12)), \
                (pos, got, want)
        if sfunc == "logsigmoid":
            s = -np.logaddexp(0.0, -s)
        np.testing.assert_allclose(z["res_s"][sl], s, rtol=1e-5, atol=1e-5)
