"""dglke_b200.emb_sim without a GPU: the flag surface against the reference's infer_emb_sim.ArgParser (recorded), the list
readers, the tile plan of every format x exec mode against a brute force, the refusals, the golden fixtures against a
float64 restatement, and the compiler log of kge_sim.cu."""
import glob
import json
import os
import re
import zlib

import numpy as np
import pytest

from emb_sim_f64 import list_keys, sim64
from predict_f64 import brute_topk

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "emb_sim")
FORMATS = ("l_r", "l_*", "*_r", "*")
MODES = ("pairwise", "all", "batch_left")


def test_flags_match_the_reference_parser():
    from dglke_b200.emb_sim import ArgParser
    want = json.load(open(os.path.join(GOLDEN, "emb_sim_flags.json")))
    got = [dict(option=a.option_strings, dest=a.dest, type=getattr(a.type, "__name__", None), default=a.default,
                nargs=a.nargs, action=type(a).__name__) for a in ArgParser()._actions if a.dest != "help"]
    assert got == want


@pytest.mark.parametrize("final_newline", [False, True])
def test_readers_take_ids_and_raw_names(tmp_path, final_newline):
    from dglke_b200.emb_sim import read_lists
    end = "\n" if final_newline else ""
    (tmp_path / "ids").write_text("3\n14\n15" + end)
    (tmp_path / "map").write_text("0\talpha\n1\tbeta\n2\tgamma\n")
    (tmp_path / "names").write_text("gamma\nalpha\ngamma" + end)
    left, right, i2e = read_lists("l_r", [str(tmp_path / "ids"), str(tmp_path / "ids")])
    assert list(left) == list(right) == [3, 14, 15] and i2e is None
    left, right, i2e = read_lists("l_*", [str(tmp_path / "names")], True, str(tmp_path / "map"))
    assert list(left) == [2, 0, 2] and right is None and i2e == {0: "alpha", 1: "beta", 2: "gamma"}
    left, right, _ = read_lists("*_r", [str(tmp_path / "names")], True, str(tmp_path / "map"))
    assert left is None and list(right) == [2, 0, 2]
    left, right, i2e = read_lists("*", None, True, str(tmp_path / "map"))
    assert left is None and right is None and i2e[1] == "beta"


@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("mode", MODES)
def test_plan_against_brute_force(fmt, mode):
    """Tiles built from the plan (left rows in batches of 3, right rows in blocks of 4) and a host merge give the brute
    force's lists, and every key decodes to its own (i, j)."""
    from dglke_b200.emb_sim import Plan
    n_rows = 11
    rng = np.random.default_rng(zlib.crc32((fmt + mode).encode()))
    nL = 5 if fmt[0] == "l" else n_rows
    nR = 7 if fmt.endswith("r") else n_rows
    if mode == "pairwise":
        if nL != nR:
            with pytest.raises(SystemExit, match="same length"):
                Plan(mode, nL, nR)
            return
    plan = Plan(mode, nL, nR)
    K = 4
    g_all, k_all = list_keys(mode, nL, nR)
    if mode == "pairwise":
        S2 = rng.permutation(nL).astype(np.float32)
        want = brute_topk(S2, g_all, k_all, plan.n_lists, K)
        i, j = plan.decode(k_all)
        assert (i == j).all() and (i == np.arange(nL)).all()
        # the pairwise tiles: [1, n] rows over consecutive pairs, key cbase + c
        sc, gr, ky = [], [], []
        for b in range(0, nL, 4):
            c = np.arange(b, min(nL, b + 4))
            sc.append(S2[c]); gr.append(np.zeros(len(c), np.int64)); ky.append(c)
    else:
        S2 = rng.permutation(nL * nR).astype(np.float32).reshape(nL, nR)
        want = brute_topk(S2.ravel(), g_all, k_all, plan.n_lists, K)
        sc, gr, ky = [], [], []
        for qb in range(0, nL, 3):
            qe = min(nL, qb + 3)
            rows, g, off = plan.queries(qb, qe)
            assert (np.diff(g) != 0).sum() == len(np.unique(g)) - 1          # a list's rows are consecutive
            for c0 in range(0, nR, 4):
                c = np.arange(c0, min(nR, c0 + 4))
                keys = off[:, None] + c[None, :] * plan.cstride
                i, j = plan.decode(keys)
                np.testing.assert_array_equal(S2[i, j], S2[rows[:, None], c[None, :]])
                sc.append(S2[rows[:, None], c[None, :]].ravel()); gr.append(np.repeat(g, len(c))); ky.append(keys.ravel())
    got = brute_topk(np.concatenate(sc), np.concatenate(gr), np.concatenate(ky), plan.n_lists, K)
    np.testing.assert_array_equal(got[1], want[1])
    np.testing.assert_array_equal(got[0], want[0])
    assert plan.n_lists == (nL if mode == "batch_left" else 1)


def test_refusals(tmp_path):
    from dglke_b200 import emb_sim
    np.save(str(tmp_path / "flat.npy"), np.zeros(10, np.float32))
    np.save(str(tmp_path / "emb.npy"), np.zeros((10, 4), np.float32))
    (tmp_path / "ids").write_text("1\n12\n")
    (tmp_path / "neg").write_text("-1\n")
    base = ["--emb_file", str(tmp_path / "emb.npy"), "--gpu", "0"]
    cases = [
        (["--format", "l_x", "--data_files", "a"] + base, "Unsupported format"),
        (["--format", "*", "--sim_func", "cos"] + base, "unknown similarity function"),
        (["--format", "*", "--exec_mode", "batch_right"] + base, "unknow execution mode"),
        (["--format", "*", "--topK", "1025"] + base, "KGE_TOPK_MAX"),
        (["--format", "*", "--topK", "0"] + base, "KGE_TOPK_MAX"),
        (["--format", "*", "--emb_file", str(tmp_path / "flat.npy"), "--gpu", "0"], "1-D"),
        (["--format", "l_*", "--data_files", str(tmp_path / "ids")] + base, "left id is outside"),
        (["--format", "*_r", "--data_files", str(tmp_path / "neg")] + base, "right id is outside"),
        (["--format", "l_*", "--data_files", str(tmp_path / "neg"), "--exec_mode", "pairwise"] + base, "left id"),
        (["--format", "l_r", "--data_files", str(tmp_path / "ids"), str(tmp_path / "ids"), "--raw_data"] + base,
         "mfile should be provided"),
        (["--format", "*"], "needs --gpu"),
        (["--format", "*", "--gpu", "0"], "emb_file should be provided"),
    ]
    for argv, msg in cases:
        with pytest.raises(SystemExit, match=msg):
            emb_sim.main(argv)
    (tmp_path / "two").write_text("1\n2\n")
    with pytest.raises(SystemExit, match="same length"):
        emb_sim.main(["--format", "l_*", "--data_files", str(tmp_path / "two"), "--exec_mode", "pairwise"] + base)
    with pytest.raises(SystemExit, match="needs 2 data files"):
        emb_sim.read_lists("l_r", [str(tmp_path / "ids")])


GOLDEN_FILES = sorted(glob.glob(os.path.join(GOLDEN, "sim_*.npz")))


def fixture_lists(z):
    emb = z["emb"]
    left = z["list_l"] if "list_l" in z else None
    right = z["list_r"] if "list_r" in z else None
    Ln = left if left is not None else np.arange(len(emb))
    Rn = right if right is not None else np.arange(len(emb))
    return emb, left, right, Ln, Rn


def test_fixture_cases_cover_every_function_mode_and_format():
    names = {os.path.basename(p) for p in GOLDEN_FILES}
    for sim in ("cosine", "l2", "l1", "dot", "ext_jaccard"):
        for mode, fmts in (("pairwise", ("l_r", "all")), ("all", ("l_r", "l_all", "all_r", "all")),
                           ("batch_left", ("l_r", "l_all", "all_r", "all"))):
            for f in fmts:
                assert "sim_%s_%s_%s.npz" % (sim, mode, f) in names
    assert {np.load(p)["emb"].shape[1] for p in GOLDEN_FILES} == {32, 41}


@pytest.mark.parametrize("path", GOLDEN_FILES, ids=lambda p: os.path.basename(p)[4:-4])
def test_fixture_against_float64(path):
    """The reference's lists are the float64 brute force's (up to exact ties -- a row against itself under l1 / l2, and
    (i, j) against (j, i) when both sides are the table -- which its argsort breaks arbitrarily), and its scores are the
    float64 scores within the fp32 bounds."""
    from dglke_b200.emb_sim import Plan
    z = np.load(path)
    mode, K, sim = str(z["exec_mode"]), int(z["k"]), str(z["sim_func"])
    emb, left, right, Ln, Rn = fixture_lists(z)
    s64, bound = sim64(sim, emb[Ln], emb[Rn], pairwise=mode == "pairwise")
    plan = Plan(mode, len(Ln), len(Rn))
    g, keys = list_keys(mode, len(Ln), len(Rn))
    ws, wk = brute_topk(s64.ravel(), g, keys, plan.n_lists, K)
    off = np.concatenate([[0], np.cumsum(z["lens"])])
    i, j = plan.decode(keys)
    score_of = dict(zip(zip(Ln[i].tolist(), Rn[j].tolist()), s64.ravel().tolist()))
    bound_of = dict(zip(zip(Ln[i].tolist(), Rn[j].tolist()), bound.ravel().tolist()))
    assert len(z["lens"]) == plan.n_lists
    for gi in range(plan.n_lists):
        m = wk[gi] >= 0
        i, j = plan.decode(wk[gi][m])
        sl = slice(off[gi], off[gi + 1])
        got = list(zip(z["res_l"][sl].tolist(), z["res_r"][sl].tolist()))
        want = list(zip(Ln[i].tolist(), Rn[j].tolist()))
        s = ws[gi][m]
        assert len(got) == len(want)
        for pos in range(len(want)):
            tie = np.isclose(s, s[pos], rtol=1e-9, atol=1e-12).sum() > 1
            assert got[pos] == want[pos] or (tie and np.isclose(score_of[got[pos]], s[pos], rtol=1e-9, atol=1e-12)), \
                (pos, got, want)
        err = np.abs(z["res_s"][sl].astype(np.float64) - np.array([score_of[p] for p in got]))
        assert (err <= np.array([bound_of[p] for p in got])).all(), (err, path)


def test_reference_self_pairs_score_negative_zero():
    """A row against itself scores exactly -0.0 under l1 / l2 in the reference: in the recorded l_* batch_left l2 CLI
    file every list starts with the query itself at -0.0."""
    lines = open(os.path.join(GOLDEN, "cli_l2.tsv")).read().split("\n")
    rows = [ln.split("\t") for ln in lines[1:-1]]
    firsts = rows[::5]
    assert all(r[0] == r[1] and r[2] == "-0.0" for r in firsts)


LOG = os.path.join(ROOT, "dgl-ke_b200", "build", "kge_sim.ptxas.log")
KERNELS = ["k_sim_prep", "k_sim_gemm", "k_sim_diffILb0", "k_sim_diffILb1", "k_sim_pairs"]


@pytest.mark.skipif(not os.path.exists(LOG), reason="no compiler log: the library was not built here")
@pytest.mark.parametrize("kernel", KERNELS)
def test_sim_kernel_compiler_log(kernel):
    """No kernel of kge_sim.cu spills, and ptxas serialises no wgmma of k_sim_gemm (C7511, C7512, C7519, C7520)."""
    log = open(LOG).read()
    blocks = re.split(r"ptxas info\s+: Compiling entry function ", log)
    hit = [b for b in blocks if b.startswith("'") and kernel in b.split("'")[1]]
    assert len(hit) == 1, "no compiler output for %s" % kernel
    assert "0 bytes spill stores, 0 bytes spill loads" in hit[0].split("Used")[0], hit[0][:400]
    for code in ("C7511", "C7512", "C7519", "C7520"):
        assert code not in log, [ln for ln in log.splitlines() if code in ln]
