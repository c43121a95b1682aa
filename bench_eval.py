"""Evaluation throughput: KEModel.forward_test against the GPU-counted ranking of dglke_b200.evaluate.

    python bench_eval.py [--edges 59071] [--big_entities 20000000] [--big_edges 100000]

Workloads (one JSON line each, plus one line naming the card and its power limit, read in the same run):
  fb15k    the FB15k shape -- TransE_l2, d = 400, 14 951 entities, 1 345 relations, 59 071 test edges x 2 sides,
           filtered by train | valid | test, every entity a candidate -- at batch_size_eval 16 and 1 000:
           forward_test (dense host bias, one rank list per batch on the host), the new path on one shard, and the new
           path on a table of two shards in this process
  sampled  a 20 M-entity table (32 GB at d = 400), 1 000 sampled candidates per chunk, batch_size_eval 1 000, filtered
The graphs are uniform random triples of those shapes (so the filter has no hub keys), tables are random.
Times are CUDA events around the whole evaluation of both sides, after a synchronise; one warm-up pass of a few batches
of every configuration runs first.  Reported: queries / s and device ms per 1 000 queries (a query = one edge, one side)."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch as th

ROOT = os.path.dirname(os.path.abspath(__file__))
for p in (ROOT, os.path.join(ROOT, "dgl-ke_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=60).stdout.strip()
        name, power = [x.strip() for x in out.split(",")]
    except Exception:
        name, power = th.cuda.get_device_name(0), "unknown"
    return {"card": name, "power_limit": power}


def timed(fn):
    th.cuda.synchronize()
    a, b = th.cuda.Event(enable_timing=True), th.cuda.Event(enable_timing=True)
    t0 = time.time()
    a.record()
    out = fn()
    b.record()
    th.cuda.synchronize()
    return a.elapsed_time(b), (time.time() - t0) * 1e3, out


def graph(n_ent, n_rel, n_train, n_valid, n_test, seed):
    rng = np.random.default_rng(seed)
    split = lambda n: tuple(rng.integers(0, m, n) for m in (n_ent, n_rel, n_ent))
    return split(n_train), split(n_valid), split(n_test)


def fb15k(args, dev, report):
    from dglke_b200.engine import DeviceTable
    from dglke_b200.evaluate import EvalSplit, Evaluator, FilterIndex, metrics_from_sums
    from dglke_b200.general_models import KEModel
    from dglke_b200.graph import TripleFilter, eval_batches
    from dglke_b200.utils import ArgParser
    n_ent, n_rel = 14951, 1345
    tr, va, te = graph(n_ent, n_rel, 483142, 50000, args.edges, 0)
    allt = tuple(np.concatenate([s[k] for s in (tr, va, te)]) for k in range(3))
    a = ArgParser().parse_args(["--gpu", "0"])
    a.eval_filter, a.strict_rel_part, a.soft_rel_part = True, False, False
    m = KEModel(a, "TransE_l2", n_ent, n_rel, 400, 19.9)
    hp = m.hyper
    known = TripleFilter(*allt, n_rel)
    split = EvalSplit(te, dev, FilterIndex.build(*allt, n_rel))
    one = m.entity_emb.table()
    half = (n_ent + 1) // 2
    e0, e1 = m.entity_emb.emb[:half].clone(), m.entity_emb.emb[half:].clone()
    two = DeviceTable([e0, e1], [th.zeros(half, device=dev), th.zeros(n_ent - half, device=dev)], n_ent, 400, [0, 0])
    n_q = 2 * args.edges

    def forward_test(batch, n=None):
        logs = []
        with th.no_grad():
            for neg_head in (True, False):
                for i, (pg, ng) in enumerate(eval_batches(*te, n_ent, batch, neg_head, known=known)):
                    if n is not None and i >= n:
                        break
                    m.forward_test(pg, ng, logs, 0)
        return {k: float(np.mean([l[k] for l in logs])) for k in logs[0]}

    def new_path(table, batch, sub=None):
        ev = Evaluator(hp, table, m.relation_emb.table(), dev)
        try:
            s = split if sub is None else sub
            return metrics_from_sums(ev.run(s, batch).cpu())
        finally:
            ev.close()

    warm = EvalSplit(tuple(x[:2000] for x in te), dev, None)
    for batch in (16, 1000):
        forward_test(batch, n=2)
        new_path(one, batch, warm)
        new_path(two, batch, warm)
        for what, fn in (("forward_test", lambda: forward_test(batch)), ("new_1_shard", lambda: new_path(one, batch)),
                         ("new_2_shards", lambda: new_path(two, batch))):
            ms, wall, met = timed(fn)
            report({"workload": "fb15k", "path": what, "batch_size_eval": batch, "queries": n_q, "device_ms": ms,
                    "wall_ms": wall, "queries_per_s": n_q / (ms / 1e3), "ms_per_1000_queries": ms / n_q * 1e3,
                    "MRR": met["MRR"], "MR": met["MR"]})


def sampled(args, dev, report):
    from dglke_b200.engine import DeviceTable, Hyper
    from dglke_b200.evaluate import EvalSplit, Evaluator, FilterIndex, metrics_from_sums
    n_ent, n_rel, d = args.big_entities, 1000, 400
    hp = Hyper(model="TransE_l2", hidden_dim=d, gamma=19.9)
    tr, va, te = graph(n_ent, n_rel, 5_000_000, 100_000, args.big_edges, 1)
    allt = tuple(np.concatenate([s[k] for s in (tr, va, te)]) for k in range(3))
    ent = th.empty((n_ent, d), device=dev).uniform_(-hp.emb_init, hp.emb_init)
    rel = th.empty((n_rel, d), device=dev).uniform_(-hp.emb_init, hp.emb_init)
    E = DeviceTable.from_tensors(ent, th.zeros(n_ent, device=dev))
    R = DeviceTable.from_tensors(rel, th.zeros(n_rel, device=dev))
    split = EvalSplit(te, dev, FilterIndex.build(*allt, n_rel))
    warm = EvalSplit(tuple(x[:4000] for x in te), dev, None)
    n_q = 2 * args.big_edges
    ev = Evaluator(hp, E, R, dev)
    try:
        ev.run(warm, 1000, 1000)
        ms, wall, acc = timed(lambda: ev.run(split, 1000, 1000).cpu())
    finally:
        ev.close()
    met = metrics_from_sums(acc)
    report({"workload": "sampled", "path": "new_1_shard", "entities": n_ent, "neg_sample_size_eval": 1000,
            "batch_size_eval": 1000, "queries": n_q, "device_ms": ms, "wall_ms": wall, "queries_per_s": n_q / (ms / 1e3),
            "ms_per_1000_queries": ms / n_q * 1e3, "MRR": met["MRR"], "MR": met["MR"]})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--edges", type=int, default=59071)
    ap.add_argument("--big_entities", type=int, default=20_000_000)
    ap.add_argument("--big_edges", type=int, default=100_000)
    ap.add_argument("--only", choices=["fb15k", "sampled"], default=None)
    args = ap.parse_args()
    if not th.cuda.is_available():
        raise SystemExit("bench_eval.py needs a CUDA device")
    dev = th.device("cuda", 0)
    th.cuda.set_device(dev)
    report = lambda d: print(json.dumps(d), flush=True)
    report(card())
    if args.only in (None, "fb15k"):
        fb15k(args, dev, report)
    if args.only in (None, "sampled"):
        sampled(args, dev, report)


if __name__ == "__main__":
    main()
