"""Link-prediction throughput: dglke_b200.predict (kge_score_neg / kge_score_pos tiles merged by kge_topk) against the
same tiles reduced by torch.topk.

    python bench_predict.py [--heads 1000] [--pairs_heads 40] [--pairs_rels 25] [--triplets 10000000]
                            [--big_entities 2500000]

Workloads (one JSON line each, plus one line naming the card and its power limit, read in the same run):
  fb15k_h**   TransE_l2, d = 400, 14 951 entities x 1 345 relations, h_*_* batch_head over --heads heads
              (1 000 x 1 345 x 14 951 = 2.0e10 scores), K = 10 and K = 1 000
  wikikg2_hr* DistMult, d = 400, a 2.5 M-entity table, h_r_* all over 1 000 (h, r) pairs (40 heads x 25 relations), K = 10
  triplets    TransE_l2 at the FB15k shape, triplet_wise over --triplets triples, K = 10
Tables and lists are random.  For each workload and K: the total time of Predictor.topk_keys (CUDA events, after one
warm-up pass), the time of the same tiles with no selection (scores only), the time of those tiles reduced by torch.topk
per list (the baseline: top-K of the tile's rows of a list, merged with the running list by a second torch.topk), and
the library's per-launch profile of one pass: milliseconds in the score kernels and in kge_topk's two kernels."""
import argparse
import json
import os
import sys

import numpy as np
import torch as th

ROOT = os.path.dirname(os.path.abspath(__file__))
for p in (ROOT, os.path.join(ROOT, "dgl-ke_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

from bench_eval import card  # noqa: E402


def _events(fn):
    th.cuda.synchronize()
    a, b = th.cuda.Event(enable_timing=True), th.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    th.cuda.synchronize()
    return a.elapsed_time(b)


def scores_only(p, plan, ids):
    for _ in p.tiles(plan, *ids):
        pass


def torch_topk(p, plan, ids, K):
    """The baseline: per tile and list, torch.topk over the list's rows, then over (running list U that)."""
    G = plan.n_lists
    run_s = th.full((G, K), float("-inf"), device=p.device)
    run_k = th.full((G, K), -1, dtype=th.int64, device=p.device)
    for S, qg, qo, cbase in p.tiles(plan, *ids):
        Q, N = S.shape
        g0, g1 = int(qg[0]), int(qg[-1])               # a list's rows are consecutive, lists ascend within a tile
        counts = th.bincount(qg - g0, minlength=g1 - g0 + 1).tolist()
        r0 = 0
        for g, n in zip(range(g0, g1 + 1), counts):
            if n == 0:
                continue
            v, i = th.topk(S[r0:r0 + n].reshape(-1), min(K, n * N))
            keys = qo[r0 + i // N] + (cbase + i % N) * plan.cstride
            v, keys = th.cat([run_s[g], v]), th.cat([run_k[g], keys])
            v2, i2 = th.topk(v, K)
            run_s[g], run_k[g] = v2, keys[i2]
            r0 += n
    return run_s, run_k


def profile(p, plan, ids, K):
    """(ms in score kernels, ms in kge_topk) over one pass, read every tile (the profiler keeps 64 records)."""
    from dglke_b200 import _lib
    G = plan.n_lists
    ts = th.full((G, K), float("-inf"), device=p.device)
    tk = th.full((G, K), -1, dtype=th.int64, device=p.device)
    p.h.profile_enable(True)
    score = topk = 0.0
    for S, qg, qo, cbase in p.tiles(plan, *ids):
        Q, N = S.shape
        _lib.check(p.lib.kge_topk(p.h.raw, S.data_ptr(), N, Q, N, qg.data_ptr(), qo.data_ptr(), cbase, plan.cstride, K,
                                  G, ts.data_ptr(), tk.data_ptr(), p.h.stream()))
        for name, ms in p.h.profile_read():
            if name.startswith("k_topk"):
                topk += ms
            else:
                score += ms
    p.h.profile_enable(False)
    return score, topk


def run(name, p, plan, ids, K, n_scores, report):
    p.topk_keys(plan, *ids, K)                     # warm-up pass: kernel loading, workspace growth
    torch_topk(p, plan, ids, K)
    total = _events(lambda: p.topk_keys(plan, *ids, K))
    base = _events(lambda: scores_only(p, plan, ids))
    tt = _events(lambda: torch_topk(p, plan, ids, K))
    sc, tp = profile(p, plan, ids, K)
    report({"workload": name, "K": K, "scores": n_scores, "total_ms": round(total, 2),
            "scores_per_s": float("%.4g" % (n_scores / total * 1e3)), "score_tiles_only_ms": round(base, 2),
            "torch_topk_total_ms": round(tt, 2), "kge_topk_over_scores_ms": round(total - base, 2),
            "torch_topk_over_scores_ms": round(tt - base, 2), "profile_score_kernels_ms": round(sc, 2),
            "profile_kge_topk_ms": round(tp, 2)})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--heads", type=int, default=1000)
    ap.add_argument("--pairs_heads", type=int, default=40)
    ap.add_argument("--pairs_rels", type=int, default=25)
    ap.add_argument("--triplets", type=int, default=10_000_000)
    ap.add_argument("--big_entities", type=int, default=2_500_000)
    args = ap.parse_args()
    from dglke_b200.engine import Hyper
    from dglke_b200.predict import Predictor, Plan
    dev = th.device("cuda", 0)
    th.cuda.set_device(dev)
    report = lambda d: print(json.dumps(d), flush=True)
    report(card())
    rng = np.random.default_rng(0)
    D, n_ent, n_rel = 400, 14951, 1345
    ids = lambda *xs: [None if x is None else th.from_numpy(np.asarray(x, np.int64)).to(dev) for x in xs]
    ent = (rng.standard_normal((n_ent, D)) * 0.05).astype(np.float32)
    rel = (rng.standard_normal((n_rel, D)) * 0.05).astype(np.float32)
    p = Predictor(Hyper(model="TransE_l2", hidden_dim=D, gamma=0.0), ent, rel, 0)
    H = rng.integers(0, n_ent, args.heads)
    plan = Plan("batch_head", len(H), n_rel, n_ent)
    for K in (10, 1000):
        run("fb15k_h**_batch_head", p, plan, ids(H, None, None), K, len(H) * n_rel * n_ent, report)
    n = args.triplets
    tri = ids(rng.integers(0, n_ent, n), rng.integers(0, n_rel, n), rng.integers(0, n_ent, n))
    run("triplet_wise", p, Plan("triplet_wise", n, n, n), tri, 10, n, report)
    p.close()
    del p
    th.cuda.empty_cache()
    big = th.empty((args.big_entities, D), dtype=th.float32, device=dev).normal_(0, 0.05)
    relb = (rng.standard_normal((500, D)) * 0.05).astype(np.float32)
    p = Predictor(Hyper(model="DistMult", hidden_dim=D, gamma=0.0), big, relb, 0)
    del big
    Hp, Rp = rng.integers(0, args.big_entities, args.pairs_heads), rng.integers(0, 500, args.pairs_rels)
    plan = Plan("all", len(Hp), len(Rp), args.big_entities)
    run("wikikg2_h_r_*_all", p, plan, ids(Hp, Rp, None), 10, len(Hp) * len(Rp) * args.big_entities, report)
    p.close()


if __name__ == "__main__":
    main()
