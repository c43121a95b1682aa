"""Generates tests/golden/emb_sim/ from the UNMODIFIED reference's EmbSimInfer.topK (models/infer.py), driven on CPU torch
through oracle/ref_harness.py's stand-ins for dgl:   python tools/gen_emb_sim_golden.py

Each sim_<function>_<mode>_<format>.npz holds the table (random), the left / right lists (absent = every row), the exec
mode, K, the function and the reference's result: the concatenated (left, right, score) columns and the length of each
list's part.  Two widths: 41 (not a multiple of 32) under the l_* and * formats, 32 under l_r and *_r.  The lists repeat
ids, and K is chosen so that some lists are shorter than K.  emb_sim_flags.json is the reference's flag table;
cli_l2.tsv is one output file of the reference's command line and cli_l2.npz its table (cli_case()).
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

OUT = os.path.join(ROOT, "tests", "golden", "emb_sim")
N_ROWS = 40
FUNCS = ("cosine", "l2", "l1", "dot", "ext_jaccard")
# exec mode -> (formats it applies to, K); pairwise needs two lists of one length
MODES = {"pairwise": (("l_r", "*"), 8), "all": (("l_r", "l_*", "*_r", "*"), 10),
         "batch_left": (("l_r", "l_*", "*_r", "*"), 9)}
LEFT = np.array([3, 17, 3, 25, 8])
RIGHT = np.array([0, 12, 12, 33, 39, 7, 20])
PAIR_LEFT, PAIR_RIGHT = np.array([3, 17, 3, 25, 8, 30]), np.array([0, 12, 12, 33, 39, 7])


def width(fmt):
    return 41 if fmt in ("l_*", "*") else 32


def table(dim, seed):
    return (np.random.default_rng(seed).standard_normal((N_ROWS, dim)) * 0.3).astype(np.float32)


def lists(mode, fmt):
    if mode == "pairwise":
        return (PAIR_LEFT, PAIR_RIGHT) if fmt == "l_r" else (None, None)
    return (LEFT if fmt[0] == "l" else None), (RIGHT if fmt.endswith("r") else None)


def flag_table():
    from dglke.infer_emb_sim import ArgParser
    return [dict(option=a.option_strings, dest=a.dest, type=getattr(a.type, "__name__", None), default=a.default,
                 nargs=a.nargs, action=type(a).__name__) for a in ArgParser()._actions if a.dest != "help"]


def main():
    rh.import_reference()
    from dglke.models.infer import EmbSimInfer
    os.makedirs(OUT, exist_ok=True)
    with open(os.path.join(OUT, "emb_sim_flags.json"), "w") as f:
        json.dump(flag_table(), f, indent=1)
    tmp = tempfile.mkdtemp(prefix="emb_sim_golden_")
    try:
        for fi, sim in enumerate(FUNCS):
            for mi, (mode, (formats, k)) in enumerate(MODES.items()):
                for xi, fmt in enumerate(formats):
                    emb = table(width(fmt), 100 * fi + 10 * mi + xi)
                    path = os.path.join(tmp, "emb.npy")
                    np.save(path, emb)
                    left, right = lists(mode, fmt)
                    inf = EmbSimInfer(-1, path, sim)
                    inf.load_emb()
                    res = inf.topK(left, right, bcast=mode == "batch_left", pair_ws=mode == "pairwise", k=k)
                    # batch_left's length-K np.full column is cut to the list's real length (zip does the same)
                    parts = [[np.asarray(c) for c in x] for x in res]
                    lens = np.array([len(p[2]) for p in parts], dtype=np.int64)
                    cols = [np.concatenate([p[c][:len(p[2])] for p in parts]) for c in range(3)]
                    name = "sim_%s_%s_%s.npz" % (sim, mode, fmt.replace("*", "all"))
                    arrays = dict(emb=emb, exec_mode=mode, fmt=fmt, k=k, sim_func=sim, lens=lens,
                                  res_l=cols[0].astype(np.int64), res_r=cols[1].astype(np.int64),
                                  res_s=cols[2].astype(np.float32))
                    for nm, x in (("list_l", left), ("list_r", right)):
                        if x is not None:
                            arrays[nm] = np.asarray(x, dtype=np.int64)
                    np.savez_compressed(os.path.join(OUT, name), **arrays)
                    print(name, lens.tolist())
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    cli_case()


CLI_LEFT = ["e3", "e17", "e25"]


def cli_case():
    """One run of the reference's command line (infer_emb_sim.main): l2, --format l_*, --exec_mode batch_left, --raw_data,
    --topK 5.  Stores the table as cli_l2.npz and the output file as cli_l2.tsv."""
    from dglke import infer_emb_sim
    emb = table(41, 999)
    tmp = tempfile.mkdtemp(prefix="emb_sim_cli_")
    try:
        np.save(os.path.join(tmp, "emb.npy"), emb)
        with open(os.path.join(tmp, "entities.dict"), "w") as f:
            f.write("".join("%d\te%d\n" % (i, i) for i in range(N_ROWS)))
        with open(os.path.join(tmp, "l.list"), "w") as f:
            f.write("".join(x + "\n" for x in CLI_LEFT))
        out = os.path.join(OUT, "cli_l2.tsv")
        argv = sys.argv
        sys.argv = ["dglke_emb_sim", "--mfile", os.path.join(tmp, "entities.dict"), "--emb_file",
                    os.path.join(tmp, "emb.npy"), "--format", "l_*", "--data_files", os.path.join(tmp, "l.list"),
                    "--raw_data", "--exec_mode", "batch_left", "--topK", "5", "--sim_func", "l2", "--output", out]
        try:
            infer_emb_sim.main()
        finally:
            sys.argv = argv
        np.savez_compressed(os.path.join(OUT, "cli_l2.npz"), emb=emb)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
