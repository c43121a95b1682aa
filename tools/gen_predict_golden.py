"""Generates tests/golden/predict/predict_*.npz from the UNMODIFIED reference's ScoreInfer.topK (models/infer.py), driven on CPU
torch through oracle/ref_harness.py's stand-ins for dgl:   python tools/gen_predict_golden.py

Each fixture holds the tables (random, so no two scores tie and the reference's argsort order is unique), the config
fields ScoreInfer reads, the H / R / T lists (absent = every entity / relation), the exec mode, K, the score function and
the reference's result: the concatenated (head, rel, tail, score) columns and the length of each list's part.
cli_DistMult.tsv is one output file of the reference's command line, cli_DistMult.npz its tables (cli_case()).
TEST INFRASTRUCTURE ONLY: it needs a checkout of the reference (KGE_REFERENCE_PY)."""
import json
import os
import shutil
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import ref_harness as rh  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "predict")
N_ENT, N_REL = 50, 7
# hidden dims: 32 and 40 put the bilinear models on both the wgmma and the fp32 tile routes of kge_score_neg
MODELS = {"TransE_l1": (32, False, False, 9.0), "TransE_l2": (40, False, False, 9.0), "DistMult": (32, False, False, 9.0),
          "ComplEx": (40, True, True, 9.0), "RESCAL": (32, False, False, 9.0), "RotatE": (40, True, False, 9.0)}
# exec mode -> (which lists are given, K)
MODES = {"triplet_wise": ("hrt", 25), "all": ("hr", 10), "batch_head": ("h", 7), "batch_rel": ("rt", 6),
         "batch_tail": ("ht", 9)}


def tables(model, seed):
    hidden, de, dr, _ = MODELS[model]
    rng = np.random.default_rng(seed)
    ed = 2 * hidden if de else hidden
    rd = 2 * hidden if dr else hidden
    if model == "RESCAL":
        rd *= ed
    ent = rng.standard_normal((N_ENT, ed)).astype(np.float32) * 0.3
    rel = rng.standard_normal((N_REL, rd)).astype(np.float32) * (0.3 if model != "RESCAL" else 0.1)
    return ent, rel


def lists(mode, seed):
    rng = np.random.default_rng(seed)
    given, _ = MODES[mode]
    if mode == "triplet_wise":
        return rng.integers(0, N_ENT, 20), rng.integers(0, N_REL, 20), rng.integers(0, N_ENT, 20)
    h = np.array([3, 17, 3, 41, 8])[: 3 if mode == "batch_head" else 5] if "h" in given else None
    r = np.array([1, 6, 2]) if "r" in given else None
    t = np.array([0, 12, 12, 33, 49, 7]) if "t" in given else None
    return h, r, t


def main():
    rh.import_reference()
    import torch as th
    from dglke.models.infer import ScoreInfer
    os.makedirs(OUT, exist_ok=True)
    tmp = tempfile.mkdtemp(prefix="predict_golden_")
    try:
        for mi, (model, (hidden, de, dr, gamma)) in enumerate(MODELS.items()):
            ent, rel = tables(model, 100 + mi)
            np.save(os.path.join(tmp, "g_%s_entity.npy" % model), ent)
            np.save(os.path.join(tmp, "g_%s_relation.npy" % model), rel)
            config = dict(model_name=model, hidden_dim=hidden, double_ent=de, double_rel=dr, gamma=gamma, dataset="g")
            for xi, (mode, (given, k)) in enumerate(MODES.items()):
                funcs = ("none", "logsigmoid") if mode in ("all", "batch_tail") else ("none",)
                for sfunc in funcs:
                    h, r, t = lists(mode, 1000 * mi + xi)
                    inf = ScoreInfer(-1, config, tmp, sfunc)
                    inf.load_model()
                    res = inf.topK(h, r, t, mode, k)
                    # the batch modes' length-K np.full column is cut to the list's real length (zip does the same)
                    parts = [[np.asarray(c) for c in x] for x in res]
                    lens = np.array([len(p[3]) for p in parts], dtype=np.int64)
                    cols = [np.concatenate([p[c][:len(p[3])] for p in parts]) for c in range(4)]
                    name = "predict_%s_%s_%s.npz" % (model, mode, sfunc)
                    arrays = dict(ent=ent, rel=rel, model=model, hidden_dim=hidden, double_ent=de, double_rel=dr,
                                  gamma=gamma, exec_mode=mode, k=k, score_func=sfunc, lens=lens,
                                  res_h=cols[0].astype(np.int64), res_r=cols[1].astype(np.int64),
                                  res_t=cols[2].astype(np.int64), res_s=cols[3].astype(np.float32))
                    for nm, x in (("list_h", h), ("list_r", r), ("list_t", t)):
                        if x is not None:
                            arrays[nm] = np.asarray(x, dtype=np.int64)
                    np.savez_compressed(os.path.join(OUT, name), **arrays)
                    print(name, lens.tolist())
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    cli_case()


CLI_LISTS = {"h": ["e3", "e17", "e41"], "t": ["e0", "e12", "e33", "e49", "e7"]}


def cli_case():
    """One run of the reference's command line (infer_score.main): DistMult, --format h_*_t, --exec_mode batch_head,
    --raw_data, --topK 5.  Stores the tables as cli_DistMult.npz and the output file as cli_DistMult.tsv."""
    from dglke import infer_score
    ent, rel = tables("DistMult", 100 + list(MODELS).index("DistMult"))
    tmp = tempfile.mkdtemp(prefix="predict_cli_")
    try:
        np.save(os.path.join(tmp, "g_DistMult_entity.npy"), ent)
        np.save(os.path.join(tmp, "g_DistMult_relation.npy"), rel)
        with open(os.path.join(tmp, "config.json"), "w") as f:
            json.dump(dict(model_name="DistMult", hidden_dim=MODELS["DistMult"][0], double_ent=False, double_rel=False,
                           gamma=MODELS["DistMult"][3], dataset="g"), f)
        for name, n in (("entities.dict", N_ENT), ("relations.dict", N_REL)):
            with open(os.path.join(tmp, name), "w") as f:
                f.write("".join("%d\t%s%d\n" % (i, name[0], i) for i in range(n)))
        for side, names in CLI_LISTS.items():
            with open(os.path.join(tmp, side + ".list"), "w") as f:
                f.write("".join(x + "\n" for x in names))
        out = os.path.join(OUT, "cli_DistMult.tsv")
        argv = sys.argv
        sys.argv = ["dglke_predict", "--model_path", tmp, "--format", "h_*_t", "--data_files",
                    os.path.join(tmp, "h.list"), os.path.join(tmp, "t.list"), "--exec_mode", "batch_head", "--raw_data",
                    "--entity_mfile", os.path.join(tmp, "entities.dict"), "--rel_mfile",
                    os.path.join(tmp, "relations.dict"), "--topK", "5", "--output", out]
        try:
            infer_score.main()
        finally:
            sys.argv = argv
        np.savez_compressed(os.path.join(OUT, "cli_DistMult.npz"), ent=ent, rel=rel)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
