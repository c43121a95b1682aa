"""Embedding-similarity throughput: dglke_b200.emb_sim (kge_sim_tile / kge_sim_pairs tiles merged by kge_topk) against torch
computing the same tiles and reducing them with torch.topk, and against kge_score_neg as the reuse route for `dot`.

    python bench_emb_sim.py [--big_rows 2500000] [--left 1000] [--pairs 10000000]

Workloads (one JSON line each, plus one line naming the card and its power limit, read in the same run):
  fb15k_*_batch_left     a 14 951 x 400 table, '*' batch_left, K = 10, each of the five functions (2.2e8 scores each)
  wikikg2_l_*_<mode>     a --big_rows x 400 table, l_* with --left left rows, all and batch_left, cosine and l2,
                         K = 10 and K = 1 000
  pairwise               --pairs random (left, right) pairs of the big table, cosine, K = 10
  reuse_*                kge_score_neg as DistMult with an all-ones relation row (scores x.y) over the same tile shapes
                         as the dot / wikikg2 dot tiles: the obvious reuse route, next to the new tile kernel's time
Per workload: the total (EmbSim.topk_keys, CUDA events, after one warm-up pass), the tile kernels alone (the same tiles
with no selection), the time kge_topk adds, torch doing the same tiles and torch.topk, achieved scores/s, and the tile
kernels' share of the binding peak: the 3xTF32 tensor rate for dot / cosine / ext_jaccard (three TF32 MMAs per
multiply-add, 2 D flops per score each, against the data sheet's 495 TFLOP/s dense TF32), the FP32 CUDA-core issue rate
for l1 / l2 (two FP32 instructions per term, against 67 TFLOP/s = 33.5 T FFMA/s).  The tile kernels' operand traffic is
far below their arithmetic at d = 400, so the arithmetic bound is the one that applies."""
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
from bench_predict import _events, scores_only  # noqa: E402

TF32_PEAK = 495e12
FP32_ISSUE = 67e12 / 2
GEMM_FUNCS = ("dot", "cosine", "ext_jaccard")


def tiles_only(s, plan, func, ids, K):
    for _ in s.tiles(plan, func, *ids, K):
        pass


def torch_tile(func, L, R):
    if func in ("l1", "l2"):
        return -th.cdist(L, R, p=1.0 if func == "l1" else 2.0)
    dot = L @ R.T
    if func == "dot":
        return dot
    nl, nr = L.norm(dim=1), R.norm(dim=1)
    if func == "cosine":
        return dot / (nl[:, None] * nr[None, :])
    return dot / (nl[:, None] ** 2 + nr[None, :] ** 2 - dot)


def torch_topk(s, plan, func, ids, K):
    """The baseline: torch computes each tile from the same rows (blocks as EmbSim sizes them), then torch.topk per list
    over (running list U the tile's part of it)."""
    Lids, Rids = ids
    rows = lambda x, b, e: s.emb[b:e, :s.dim] if x is None else s.emb[x[b:e], :s.dim]
    if plan.mode == "pairwise":
        run = th.full((K,), float("-inf"), device=s.device)
        nb = 1 << 22
        for b in range(0, plan.nL, nb):
            e = min(plan.nL, b + nb)
            L, R = rows(Lids, b, e), rows(Rids, b, e)
            if func == "cosine":
                v = (L * R).sum(1) / (L.norm(dim=1) * R.norm(dim=1))
            else:
                v = torch_tile(func, L, R).diagonal()
            run = th.topk(th.cat([run, v]), K).values
        return
    Qb = min(plan.nL, s.query_batch)
    nb = min(plan.nR, s.block_rows(Qb, K))
    run_all = th.full((K,), float("-inf"), device=s.device)
    for qb in range(0, plan.nL, Qb):
        qe = min(plan.nL, qb + Qb)
        L = rows(Lids, qb, qe)
        run = th.full((qe - qb, K), float("-inf"), device=s.device)
        for c0 in range(0, plan.nR, nb):
            S = torch_tile(func, L, rows(Rids, c0, min(plan.nR, c0 + nb)))
            if plan.mode == "batch_left":
                run = th.topk(th.cat([run, th.topk(S, min(K, S.shape[1]), dim=1).values], 1), K, dim=1).values
            else:
                run_all = th.topk(th.cat([run_all, th.topk(S.reshape(-1), min(K, S.numel())).values]), K).values


def run(name, s, plan, func, ids, K, report):
    n_scores = plan.nL if plan.mode == "pairwise" else plan.nL * plan.nR
    s.topk_keys(plan, func, *ids, K)                     # warm-up pass: kernel loading, workspace growth
    torch_topk(s, plan, func, ids, K)
    total = _events(lambda: s.topk_keys(plan, func, *ids, K))
    tiles = _events(lambda: tiles_only(s, plan, func, ids, K))
    tt = _events(lambda: torch_topk(s, plan, func, ids, K))
    D = s.dim
    if plan.mode == "pairwise":
        bound, share = "memory (pairs)", None
    elif func in GEMM_FUNCS:
        bound, share = "3xTF32 tensor", 3 * 2 * D * n_scores / (tiles * 1e-3) / TF32_PEAK
    else:
        bound, share = "FP32 CUDA-core", 2 * D * n_scores / (tiles * 1e-3) / FP32_ISSUE
    report({"workload": name, "sim_func": func, "K": K, "scores": n_scores, "total_ms": round(total, 2),
            "scores_per_s": float("%.4g" % (n_scores / total * 1e3)), "tile_kernels_ms": round(tiles, 2),
            "kge_topk_adds_ms": round(total - tiles, 2), "torch_tiles_and_topk_ms": round(tt, 2),
            "tile_scores_per_s": float("%.4g" % (n_scores / tiles * 1e3)), "binding_peak": bound,
            "tile_share_of_peak": None if share is None else round(share, 3)})


def reuse(name, emb, n_left, report):
    """kge_score_neg DistMult with an all-ones relation: the dot scores of n_left query rows against the whole table, in
    Predictor's tiles (the same query batch of 2 048 and the same workspace budget)."""
    from dglke_b200.engine import Hyper
    from dglke_b200.predict import Predictor, Plan
    D = emb.shape[1]
    p = Predictor(Hyper(model="DistMult", hidden_dim=D, gamma=0.0), emb, np.ones((1, D), np.float32), 0)
    try:
        plan = Plan("batch_head", n_left, 1, emb.shape[0])
        ids = [th.arange(n_left, device=p.device), None, None]
        scores_only(p, plan, ids)
        t = _events(lambda: scores_only(p, plan, ids))
    finally:
        p.close()
    n = n_left * emb.shape[0]
    report({"workload": name, "route": "kge_score_neg DistMult, relation = ones", "scores": n,
            "tile_kernels_ms": round(t, 2), "tile_scores_per_s": float("%.4g" % (n / t * 1e3)),
            "tile_share_of_peak": round(3 * 2 * D * n / (t * 1e-3) / TF32_PEAK, 3)})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--big_rows", type=int, default=2_500_000)
    ap.add_argument("--left", type=int, default=1000)
    ap.add_argument("--pairs", type=int, default=10_000_000)
    args = ap.parse_args()
    from dglke_b200.emb_sim import EmbSim, Plan
    dev = th.device("cuda", 0)
    th.cuda.set_device(dev)
    report = lambda d: print(json.dumps(d), flush=True)
    report(card())
    rng = np.random.default_rng(0)
    D, n = 400, 14951
    emb = (rng.standard_normal((n, D)) * 0.05).astype(np.float32)
    s = EmbSim(emb, 0)
    plan = Plan("batch_left", n, n)
    for func in ("dot", "cosine", "ext_jaccard", "l2", "l1"):
        run("fb15k_*_batch_left", s, plan, func, [None, None], 10, report)
    s.close()
    reuse("reuse_fb15k_dot", emb, n, report)
    del s
    th.cuda.empty_cache()
    big = th.empty((args.big_rows, D), dtype=th.float32, device=dev).normal_(0, 0.05)
    s = EmbSim(big, 0)
    left = th.from_numpy(rng.integers(0, args.big_rows, args.left)).to(dev)
    for mode in ("all", "batch_left"):
        plan = Plan(mode, args.left, args.big_rows)
        for func in ("cosine", "l2"):
            for K in (10, 1000):
                run("wikikg2_l_*_" + mode, s, plan, func, [left, None], K, report)
    plan = Plan("batch_left", args.left, args.big_rows)
    run("wikikg2_l_*_batch_left", s, plan, "dot", [left, None], 10, report)
    pl = th.from_numpy(rng.integers(0, args.big_rows, args.pairs)).to(dev)
    pr = th.from_numpy(rng.integers(0, args.big_rows, args.pairs)).to(dev)
    run("pairwise", s, Plan("pairwise", args.pairs, args.pairs), "cosine", [pl, pr], 10, report)
    s.close()
    del s
    th.cuda.empty_cache()
    reuse("reuse_wikikg2_dot", big[:args.big_rows].cpu().numpy(), args.left, report)


if __name__ == "__main__":
    main()
