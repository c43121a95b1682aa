"""Evaluation on the sharded entity table with two ranks, launched with torchrun (see tests/test_gpu_eval_sharded.py):

    torchrun --nproc-per-node 2 tests/dist_eval_check.py

A few pipelined training steps (each step announces the next, kge_set_next_batch), a validation between two of them,
more steps, then a test over both ranks' slices.  The pooled test sums must equal a one-process evaluation of the same
edges on the gathered table, and count 2 x the edges (both corruption sides).  TransE_l2 trains on the fused kernels,
which stage the next step's rows; evaluation batches of 13 queries keep every score tile off the wgmma engine (13, 10, 11
or 8 queries against 2 001, 2 000 or 4 001 rows), so the gathered one-shard table and the two shards give bitwise equal
scores and the ranks agree exactly.

DIST_SAME_GPU=1 puts both ranks on cuda:0 with the gloo backend, as tests/dist_check.py does."""
import os
import sys

import numpy as np
import torch as th
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "dgl-ke_b200"), os.path.join(ROOT, "oracle")):
    sys.path.insert(0, p)


def main():
    from dglke_b200.engine import Hyper, DeviceTable
    from dglke_b200.dist import ShardedTrainer
    from dglke_b200.evaluate import EvalSplit, Evaluator, FilterIndex, metrics_from_sums

    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    same_gpu = os.environ.get("DIST_SAME_GPU") == "1"
    local = 0 if same_gpu else int(os.environ["LOCAL_RANK"])
    th.cuda.set_device(local)
    dev = th.device("cuda", local)
    if same_gpu:
        dist.init_process_group("gloo")
    else:
        dist.init_process_group("nccl", device_id=dev)
    n_ent, n_rel, B, N = 4001, 16, 256, 64
    hp = Hyper(model="TransE_l2", hidden_dim=64, gamma=12.0, lr=0.2, reg_coef=1e-6, adversarial=True)
    tr = ShardedTrainer(hp, n_ent, n_rel, dev, seed=1)
    g = np.random.default_rng(0)                   # the same graph on every rank
    train = tuple(g.integers(0, m, 3000) for m in (n_ent, n_rel, n_ent))
    valid = tuple(g.integers(0, m, 101) for m in (n_ent, n_rel, n_ent))
    test = tuple(g.integers(0, m, 203) for m in (n_ent, n_rel, n_ent))
    index = FilterIndex.build(*(np.concatenate([s[k] for s in (train, valid, test)]) for k in range(3)), n_rel)
    vsplit = EvalSplit(valid, dev, index, rank, world)
    tsplit = EvalSplit(test, dev, index, rank, world)

    steps, batches = 5, []
    for s in range(steps):
        rng = np.random.default_rng(1000 * rank + s)
        e = rng.integers(0, 3000, B)
        h, r, t = train[0][e], train[1][e], train[2][e]
        nodes, inv = np.unique(np.concatenate([h, t]), return_inverse=True)
        T = lambda a: th.from_numpy(np.ascontiguousarray(a.astype(np.int64))).to(dev)
        batches.append([T(nodes), T(inv[:B]), T(inv[B:]), T(r), T(rng.integers(0, n_ent, B))])
    launches = []
    for s in range(steps):
        nxt = (batches[s + 1][0], batches[s + 1][4]) if 0 < s + 1 < steps - 1 else None
        n0 = tr.h.launch_count()
        tr.step(*batches[s], N, N, bool(s % 2), next_batch=nxt)
        launches.append(tr.h.launch_count() - n0)
        if s == 1:                                  # step 2 is announced: its rows are staged across the validation
            local_sums, pooled = tr.evaluate(vsplit, 13)
            assert float(local_sums[5]) == 2 * vsplit.n and float(pooled[5]) == 2 * 101, (local_sums, pooled)
            print("[{}]Valid average MRR: {}".format(rank, metrics_from_sums(local_sums)["MRR"]), flush=True)
    assert launches[1] == launches[2] == launches[3] == launches[4] - 1, "staged rows were not used: %r" % (launches,)
    tr.barrier()
    _, pooled = tr.evaluate(tsplit, 13)
    full = tr.gather_entity_table()
    assert bool(th.isfinite(full).all())
    if rank == 0:
        one = DeviceTable.from_tensors(full.contiguous(), th.zeros(n_ent, device=dev))
        ev = Evaluator(hp, one, tr.rel, dev)
        try:
            ref = ev.run(EvalSplit(test, dev, index), 13).cpu()
        finally:
            ev.close()
        assert float(pooled[5]) == 2 * 203, pooled
        for i in range(1, 6):
            assert float(pooled[i]) == float(ref[i]), (i, pooled.tolist(), ref.tolist())
        assert abs(float(pooled[0]) - float(ref[0])) <= 1e-12 * float(ref[0]), (pooled.tolist(), ref.tolist())
        print("DIST_EVAL_OK world=%d %s" % (world, metrics_from_sums(pooled)), flush=True)
    dist.barrier()
    tr.close()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
