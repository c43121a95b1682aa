"""dglke_train-compatible entry point (reference: train.py:74-380, train_pytorch.py:110-197).

    python -m dglke_b200.train --model_name TransE_l2 --dataset FB15k --batch_size 1000 \
        --neg_sample_size 200 --hidden_dim 400 --gamma 19.9 --lr 0.25 --max_step 24000 -adv --gpu 0

All reference flags parse.  What differs, and why:
  * data: the reference's on-disk formats are read by dglke_b200.dataset (built-in layouts when they are unpacked under
    --data_path, udd_{hrt..} integer files, raw_udd_{hrt..} string files whose dictionaries get built).  There is no
    network in this environment: a built-in dataset that is not on disk selects the dataset's SHAPE (entities /
    relations / training edges) and the triples are drawn synthetically;
  * --gpu is required (no CPU path).  One GPU id: one process, KEModel over the fused 5-kernel step.  Several ids
    (`--gpu 0 1 2 3`, the reference's multi-GPU spelling, train.py:290-317): one process per GPU is spawned, the entity
    table is row-sharded over the GPUs' HBM (replacing --mix_cpu_gpu's host table) and trained through
    dglke_b200.dist.ShardedTrainer (peer loads / red.add over NVLink, NCCL all-reduce of the relation gradients);
  * sampling runs on the GPU (dglke_b200.sampler.DeviceSampler replaces DGL's C++ EdgeSampler; --host_sampler selects
    the numpy samplers of dglke_b200.graph instead).
"""
import os
import sys
import time

import numpy as np
import torch as th

from .utils import ArgParser, get_compatible_batch_size, save_model, save_config, prepare_save_path
from .general_models import KEModel
from .graph import SyntheticSampler, TripleSampler, TripleFilter, eval_batches, NegGraph
from .sampler import DeviceSampler
from .evaluate import EvalSplit, Evaluator, FilterIndex, check_eval_flags, metrics_from_sums, select_eval_edges

# (entities, relations, training edges): docs/source/benchmarks.rst dataset table
BUILTIN_SHAPES = {
    "FB15k": (14951, 1345, 483142), "FB15k-237": (14541, 237, 272115), "wn18": (40943, 18, 141442),
    "wn18rr": (40943, 11, 86835), "Freebase": (86054151, 14824, 304727650),
    "wikikg2": (2500604, 535, 16109182), "biokg": (93773, 51, 4762678),
}


def _load_dataset(args):
    """train.py:62-116 of the reference: get_dataset(data_path, dataset, format, delimiter, data_files,
    has_edge_importance).  Returns (n_entities, n_relations, train, valid, test, dataset or None); a built-in dataset that
    is not on disk (there is no network here) becomes a synthetic graph of its published shape."""
    from .dataset import get_dataset
    if args.format == "built_in" and args.dataset in BUILTIN_SHAPES:
        try:
            ds = get_dataset(args.data_path, args.dataset, "built_in")
        except (FileNotFoundError, NotImplementedError) as e:
            n_ent, n_rel, n_edges = BUILTIN_SHAPES[args.dataset]
            print("NOTE: %s\nNOTE: training on a synthetic graph of %s's shape (%d entities, %d relations)" % (
                e, args.dataset, n_ent, n_rel))
            return n_ent, n_rel, None, None, None, None
    else:
        ds = get_dataset(args.data_path, args.dataset, args.format, args.delimiter, args.data_files,
                         getattr(args, "has_edge_importance", False))
    return ds.n_entities, ds.n_relations, ds.train, ds.valid, ds.test, ds


class _DevicePosGraph:
    """What KEModel.forward needs from a device-sampled batch: the kge_batch_t itself."""

    def __init__(self, batch):
        self.device_batch = batch
        self.ndata, self.edata = {}, {}

    def number_of_edges(self):
        return self.device_batch.B


class DeviceGraphSampler:
    """Iterator of (pos_g, neg_g) over dglke_b200.sampler.DeviceSampler (same protocol as the numpy samplers)."""

    def __init__(self, heads, rels, tails, n_entities, batch_size, neg_sample_size, seed=0, device=0):
        self.s = DeviceSampler(heads, rels, tails, n_entities, batch_size, neg_sample_size, seed=seed, device=device)
        self.k = 0

    def __iter__(self):
        return self

    def __next__(self):
        b = self.s.sample(self.k)
        self.k += 1
        dummy = th.empty(0, dtype=th.int64)
        ng = NegGraph(dummy, self.s.num_chunks, self.s.chunk_size, self.s.Ns, b.neg_head)
        return _DevicePosGraph(b), ng


def synthetic_edges(n_ent, n_rel, n_edges, seed=0):
    """A synthetic training graph of a built-in dataset's shape (there is no network to download the real one)."""
    rng = np.random.default_rng(seed)
    n_edges = int(min(n_edges, 20_000_000))
    return rng.integers(0, n_ent, n_edges), rng.integers(0, n_rel, n_edges), rng.integers(0, n_ent, n_edges)


def train(args, model, train_sampler, valid_batches=None, rank=0, barrier=None):
    """train_pytorch.py:110-197 -- same four phases and the same log lines."""
    gpu_id = args.gpu[rank % len(args.gpu)]
    logs = []
    train_start = start = time.time()
    sample_time = update_time = forward_time = backward_time = 0.0
    for step in range(0, args.max_step):
        t0 = time.time()
        pos_g, neg_g = next(train_sampler)
        sample_time += time.time() - t0
        t0 = time.time()
        loss, log = model.forward(pos_g, neg_g, gpu_id)
        forward_time += time.time() - t0
        t0 = time.time()
        loss.backward()
        backward_time += time.time() - t0
        t0 = time.time()
        model.update(gpu_id)
        update_time += time.time() - t0
        logs.append(log)
        if args.force_sync_interval > 0 and (step + 1) % args.force_sync_interval == 0 and barrier is not None:
            barrier()
        if (step + 1) % args.log_interval == 0:
            th.cuda.synchronize()
            for k in logs[0].keys():
                v = sum(l[k] for l in logs) / len(logs)
                print("[proc {}][Train]({}/{}) average {}: {}".format(rank, (step + 1), args.max_step, k, v))
            logs = []
            print("[proc {}][Train] {} steps take {:.3f} seconds".format(rank, args.log_interval, time.time() - start))
            print("[proc {}]sample: {:.3f}, forward: {:.3f}, backward: {:.3f}, update: {:.3f}".format(
                rank, sample_time, forward_time, backward_time, update_time))
            sample_time = update_time = forward_time = backward_time = 0.0
            start = time.time()
        if args.valid and (step + 1) % args.eval_interval == 0 and step > 1 and valid_batches is not None:
            test(args, model, valid_batches(), rank, mode="Valid")
    th.cuda.synchronize()
    print("proc {} takes {:.3f} seconds".format(rank, time.time() - train_start))


def test(args, model, batches, rank=0, mode="Test"):
    """train_pytorch.py:199-253 (non-wikikg90M branch): average MRR / MR / HITS@k over head and tail ranking."""
    gpu_id = args.gpu[rank % len(args.gpu)]
    if isinstance(batches, EvalSplit):
        # --neg_sample_size_eval > 0: chunked sampled candidates, ranks counted on the GPU (dglke_b200.evaluate)
        ev = Evaluator(model.hyper, model.entity_emb.table(), model.relation_emb.table(), model.device)
        try:
            metrics = metrics_from_sums(ev.run(batches, args.batch_size_eval, args.neg_sample_size_eval).cpu())
        finally:
            ev.close()
    else:
        logs = []
        with th.no_grad():
            for pos_g, neg_g in batches:
                model.forward_test(pos_g, neg_g, logs, gpu_id)
        metrics = {}
        if logs:
            for m in logs[0].keys():
                metrics[m] = sum(l[m] for l in logs) / len(logs)
    for k, v in metrics.items():
        print("[{}]{} average {}: {}".format(rank, mode, k, v))
    return metrics


def main(argv=None):
    args = ArgParser().parse_args(argv)
    if args.gpu[0] < 0:
        raise SystemExit("dglke_b200 needs --gpu: the hot path is an H100 CUDA library without a CPU fallback")
    check_eval_flags(args)
    prepare_save_path(args)
    args.eval_filter = not args.no_eval_filter
    args.strict_rel_part = args.soft_rel_part = False
    args.batch_size = get_compatible_batch_size(args.batch_size, args.neg_sample_size)
    args.batch_size_eval = get_compatible_batch_size(args.batch_size_eval, args.neg_sample_size_eval)
    n_ent, n_rel, tr, va, te, dataset = _load_dataset(args)
    n_edges = BUILTIN_SHAPES[args.dataset][2] if tr is None else len(tr[0])
    if dataset is not None:
        print("|Train|: {}  entities: {}  relations: {}".format(len(tr[0]), n_ent, n_rel))
    if tr is not None and len(tr) == 4 and not args.has_edge_importance:
        tr = tr[:3]
    # filtered evaluation (the default; --no_eval_filter turns it off): candidates that form a triple of train / valid /
    # test are left out of the ranking (EvalDataset builds its graph from all three splits, sampler.py:604-640)
    known_triples = None
    if args.eval_filter and dataset is not None and (va is not None or te is not None):
        allt = [x for x in (tr, va, te) if x is not None]
        known_triples = tuple(np.concatenate([x[k] for x in allt]) for k in range(3))
    va, te = (None if s is None else select_eval_edges(s, args.eval_percent, seed=k) for k, s in enumerate((va, te)))
    if len(args.gpu) > 1:
        return train_multi_gpu(args, n_ent, n_rel, tr if tr is not None else synthetic_edges(n_ent, n_rel, n_edges),
                               va, te, known_triples)
    th.cuda.set_device(args.gpu[0])
    model = KEModel(args, args.model_name, n_ent, n_rel, args.hidden_dim, args.gamma,
                    double_entity_emb=args.double_ent, double_relation_emb=args.double_rel)
    host = getattr(args, "host_sampler", False) or args.has_edge_importance
    if host and tr is None:
        sampler = SyntheticSampler(n_ent, n_rel, args.batch_size, args.neg_sample_size, seed=0)
    elif host:
        sampler = TripleSampler(tr[0], tr[1], tr[2], n_ent, n_rel, args.batch_size, args.neg_sample_size, seed=0,
                                impts=tr[3] if len(tr) == 4 else None)
    else:
        edges = tr if tr is not None else synthetic_edges(n_ent, n_rel, n_edges)
        sampler = DeviceGraphSampler(edges[0], edges[1], edges[2], n_ent, args.batch_size, args.neg_sample_size, seed=0,
                                     device=args.gpu[0])

    known = index = None
    if known_triples is not None and args.neg_sample_size_eval > 0:
        index = FilterIndex.build(*known_triples, n_rel)
    elif known_triples is not None:
        known = TripleFilter(*known_triples, n_rel)

    def split_batches(split):
        if args.neg_sample_size_eval > 0:
            es = EvalSplit(split, model.device, index)
            return lambda: es

        def gen():
            for neg_head in (True, False):
                yield from eval_batches(split[0], split[1], split[2], n_ent, args.batch_size_eval, neg_head, known=known)
        return gen
    train(args, model, sampler, split_batches(va) if (args.valid and va is not None) else None)
    if not args.no_save_emb:
        save_model(args, model)
    if args.test and te is not None:
        test(args, model, split_batches(te)())
    return model


def hyper_from_args(args):
    """The step hyper-parameters of the parsed command line: every field of engine.Hyper, the loss flags included."""
    from .engine import Hyper
    return Hyper(model=args.model_name, hidden_dim=args.hidden_dim, gamma=args.gamma, lr=args.lr,
                 reg_coef=args.regularization_coef, reg_norm=args.regularization_norm,
                 adversarial=args.neg_adversarial_sampling, adv_temperature=args.adversarial_temperature,
                 double_ent=args.double_ent, double_rel=args.double_rel, loss_genre=args.loss_genre,
                 margin=args.margin, pairwise=args.pairwise, neg_deg_sample=args.neg_deg_sample)


def _multi_gpu_worker(rank, world, args, n_ent, n_rel, edges, port, valid=None, test=None, index=None):
    """One process per GPU (reference: train.py:298-317 forks one process per GPU over a shared host table).
    valid / test: the evaluation splits (after --eval_percent); index: evaluate.FilterIndex of the known triples, or None
    (raw ranks).  Rank r evaluates its slice of each split (evaluate.rank_slice)."""
    import torch.distributed as dist
    from .dist import ShardedTrainer
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    dev = th.device("cuda", args.gpu[rank])
    th.cuda.set_device(dev)
    dist.init_process_group("nccl", device_id=dev)
    trainer = ShardedTrainer(hyper_from_args(args), n_ent, n_rel, dev, seed=0)
    # edge partition: the edges whose head row this rank owns (half of the positive-node traffic stays on the GPU);
    # KGE_B200_EDGE_PART=random gives the reference's RandomPartition (dataloader/sampler.py:256-290)
    if os.environ.get("KGE_B200_EDGE_PART", "head_owner") == "random":
        perm = np.random.default_rng(0).permutation(len(edges[0]))[rank::world]
    else:
        from .dist import partition_edges_by_head_owner
        perm = partition_edges_by_head_owner(edges[0], n_ent, world, rank)
        if len(perm) < args.batch_size:
            raise SystemExit("rank %d owns the heads of only %d edges (< batch_size): use KGE_B200_EDGE_PART=random" % (rank, len(perm)))
    sampler = DeviceSampler(edges[0][perm], edges[1][perm], edges[2][perm], n_ent, args.batch_size, args.neg_sample_size,
                            seed=1000 + rank, device=dev.index)
    vsplit = EvalSplit(valid, dev, index, rank, world) if args.valid and valid is not None else None
    tsplit = EvalSplit(test, dev, index, rank, world) if args.test and test is not None else None
    start = t0 = time.time()
    logs = []
    # --async_update (tensor_models.py:136-175: the update runs behind the trainer, which may read rows one update old):
    # the sampler runs one batch ahead and the fused kernels of step k fetch the rows of step k+1 over NVLink while they
    # compute (kge_set_next_batch); without the flag every step gathers its own, fully up-to-date rows
    pipelined = bool(getattr(args, "async_update", False))
    ahead = sampler.sample(0) if pipelined else None
    for step in range(args.max_step):
        if pipelined:
            b, ahead = ahead, sampler.sample(step + 1)      # the sampler's output buffers alternate: both batches stay valid
        else:
            b = sampler.sample(step)
        log4 = trainer.step(b, chunk_size=sampler.chunk_size, neg_sample_size=args.neg_sample_size, next_batch=ahead)
        if (step + 1) % args.log_interval == 0:
            v = log4.cpu().tolist()
            print("[proc {}][Train]({}/{}) average loss: {} (pos {}, neg {}, reg {})".format(rank, step + 1, args.max_step, v[2],
                                                                                      v[0], v[1], v[3]))
            print("[proc {}][Train] {} steps take {:.3f} seconds".format(rank, args.log_interval, time.time() - start))
            start = time.time()
        if args.force_sync_interval > 0 and (step + 1) % args.force_sync_interval == 0:
            trainer.barrier()                       # train_pytorch.py:157-159
        if vsplit is not None and (step + 1) % args.eval_interval == 0 and step > 1:
            # between step k and k+1: a step announced with --async_update keeps the rows staged for it
            local, _ = trainer.evaluate(vsplit, args.batch_size_eval, args.neg_sample_size_eval)
            for k, v in metrics_from_sums(local).items():
                print("[{}]Valid average {}: {}".format(rank, k, v))
    trainer.barrier()
    print("proc {} takes {:.3f} seconds".format(rank, time.time() - t0))
    if tsplit is not None:
        _, pooled = trainer.evaluate(tsplit, args.batch_size_eval, args.neg_sample_size_eval)
        if rank == 0:                               # train.py:357-369: the ranks of every process, pooled
            print("-------------- Test result --------------")
            for k, v in metrics_from_sums(pooled).items():
                print("Test average {} : {}".format(k, v))
            print("-----------------------------------------")
    if not args.no_save_emb:
        ent = trainer.gather_entity_table()
        if rank == 0:
            os.makedirs(args.save_path, exist_ok=True)
            name = args.dataset + "_" + args.model_name
            np.save(os.path.join(args.save_path, name + "_entity.npy"), ent.cpu().numpy())
            np.save(os.path.join(args.save_path, name + "_relation.npy"), trainer.rel_emb.cpu().numpy())
            save_config(args)
    dist.barrier()
    dist.destroy_process_group()


def train_multi_gpu(args, n_ent, n_rel, edges, valid=None, test=None, known_triples=None):
    import torch.multiprocessing as mp
    world = len(args.gpu)
    if args.has_edge_importance:
        raise SystemExit("--has_edge_importance is single-GPU only here")
    if args.neg_deg_sample:
        raise SystemExit("--neg_deg_sample is single-GPU only here: it needs an unsharded entity table")
    port = 29400 + os.getpid() % 1000
    edges = tuple(np.ascontiguousarray(e, dtype=np.int64) for e in edges)
    index = FilterIndex.build(*known_triples, n_rel) if known_triples is not None and (args.valid or args.test) else None
    mp.spawn(_multi_gpu_worker, args=(world, args, n_ent, n_rel, edges, port, valid, test, index), nprocs=world, join=True)
    return None


if __name__ == "__main__":
    main()
