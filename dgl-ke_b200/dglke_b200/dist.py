"""Single-box multi-GPU training: one process per GPU (torch.distributed, NCCL).

Replaces the reference's multi-GPU data flow (--mix_cpu_gpu: entity table in host shared memory,
H2D gather / D2H scatter per step, train.py:92-95, tensor_models.py:292-294,330-361) with:

  * entity table + Adagrad state: contiguous row-range shards, one per GPU's HBM
    (owner(id) = id // ceil(N_e / G)); every rank maps all peers' shards (CUDA virtual-memory allocations passed
    between the ranks as file descriptors: 2 MiB pages on both sides -- a cudaIpc mapping of a 69 GB shard is
    TLB-miss bound, 6x slower), so the step kernels gather remote rows with peer loads and scatter updates with
    system-scope red.add over NVLink / NVSwitch from inside the kernel -- no entity collective;
  * edges: data parallel, each rank trains on its own edge stream (reference: RandomPartition,
    dataloader/sampler.py:256-290), Hogwild across GPUs as the reference is across processes;
  * relation table: replicated; per-relation gradient sums and mean(g^2) sums are all-reduced with
    NCCL every step and every replica applies the identical Adagrad update (the only collective).
"""
import ctypes as C
import os
import socket

import torch
import torch.distributed as dist

from . import _lib
from .engine import StepEngine, DeviceTable


class _ExternalBuffer:
    """Wraps a raw device pointer as a torch tensor through __cuda_array_interface__."""

    def __init__(self, ptr, shape):
        self.__cuda_array_interface__ = {"shape": tuple(shape), "typestr": "<f4", "data": (int(ptr), False),
                                         "version": 3, "strides": None}


def exchange_fds(fds, rank, world, group=None):
    """Every rank hands its file descriptors to every peer over Unix sockets (SCM_RIGHTS).  Returns
    {peer_rank: [fd, ...]} for the peers; the caller closes what it receives after mapping."""
    token = [os.urandom(8).hex() if rank == 0 else None]
    dist.broadcast_object_list(token, src=0, group=group)
    name = lambda r: "\0kge_b200_%s_%d" % (token[0], r)                # abstract namespace: nothing to unlink
    srv = socket.socket(socket.AF_UNIX, socket.SOCK_STREAM)
    srv.bind(name(rank))
    srv.listen(world)
    dist.barrier(group=group)                                          # every rank is listening
    for peer in range(world):
        if peer == rank:
            continue
        with socket.socket(socket.AF_UNIX, socket.SOCK_STREAM) as c:
            c.connect(name(peer))
            socket.send_fds(c, [rank.to_bytes(4, "little")], list(fds))
    got = {}
    for _ in range(world - 1):
        conn, _addr = srv.accept()
        with conn:
            msg, rfds, _flags, _a = socket.recv_fds(conn, 4, len(fds))
            assert len(rfds) == len(fds), "short descriptor message"
            got[int.from_bytes(msg, "little")] = rfds
    srv.close()
    dist.barrier(group=group)
    return got


def shard_rows(num_rows, world, rank):
    per = (num_rows + world - 1) // world
    lo = min(num_rows, rank * per)
    hi = min(num_rows, (rank + 1) * per)
    return per, lo, hi


def owner_of(ids, num_rows, world):
    per = (num_rows + world - 1) // world
    return ids // per


def partition_edges_by_head_owner(heads, n_ent, world, rank):
    """Indices of the edges whose HEAD row lives in `rank`'s shard.  With this edge partition half of a batch's
    positive-node rows are local (gather and Adagrad scatter stay on the GPU); the reference's analogue is its partitioned
    training, where a trainer's edges are those whose entities are mostly local (METIS, partition.py / RandomPartition
    keeps no locality at all).  Every edge still belongs to exactly one rank."""
    import numpy as np
    per = (n_ent + world - 1) // world
    return np.nonzero(np.asarray(heads) // per == rank)[0]


class ShardedTrainer:
    """StepEngine-compatible driver (step / step_host / sync / h) over a sharded entity table."""

    def __init__(self, hp, n_ent, n_rel, device, seed=0, group=None):
        self.hp, self.device, self.group = hp, device, group
        self.world = dist.get_world_size(group)
        self.rank = dist.get_rank(group)
        self.h = _lib.get_handle(device.index)
        lib = self.h.lib
        De, Dr = hp.entity_dim, hp.relation_dim
        per, lo, hi = shard_rows(n_ent, self.world, self.rank)
        assert hi > lo, "more GPUs than entity rows"
        self.n_ent, self.n_rel, self.rows_per_shard, self.row_lo, self.row_hi = n_ent, n_rel, per, lo, hi
        # local shard: shareable VMM allocation (kge_shard_alloc); every shard has the size of a full one so that the
        # importers know it
        n_local = hi - lo
        emb_bytes, st_bytes = per * De * 4, max(per, 1) * 4
        p_emb, p_st = C.c_void_p(), C.c_void_p()
        fd_emb, fd_st = C.c_int(-1), C.c_int(-1)
        _lib.check(lib.kge_shard_alloc(self.h.raw, emb_bytes, C.byref(p_emb), C.byref(fd_emb)))
        _lib.check(lib.kge_shard_alloc(self.h.raw, st_bytes, C.byref(p_st), C.byref(fd_st)))
        self._owned = [(p_emb.value, emb_bytes), (p_st.value, st_bytes)]
        self.ent_local = torch.as_tensor(_ExternalBuffer(p_emb.value, (n_local, De)), device=device)
        self.ent_state_local = torch.as_tensor(_ExternalBuffer(p_st.value, (n_local,)), device=device)
        g = torch.Generator(device=device).manual_seed(seed * 1000003 + self.rank)
        self.ent_local.uniform_(-hp.emb_init, hp.emb_init, generator=g)
        self.ent_state_local.zero_()
        peers = exchange_fds([fd_emb.value, fd_st.value], self.rank, self.world, group)
        os.close(fd_emb.value)
        os.close(fd_st.value)
        emb_ptrs, st_ptrs = [], []
        for r in range(self.world):
            if r == self.rank:
                emb_ptrs.append(p_emb.value)
                st_ptrs.append(p_st.value)
                continue
            ptrs = []
            for fd, nbytes in zip(peers[r], (emb_bytes, st_bytes)):
                out = C.c_void_p()
                _lib.check(lib.kge_shard_import(self.h.raw, fd, nbytes, C.byref(out)))
                os.close(fd)
                ptrs.append(out.value)
                self._owned.append((out.value, nbytes))
            emb_ptrs.append(ptrs[0])
            st_ptrs.append(ptrs[1])
        self.ent = DeviceTable(emb_ptrs, st_ptrs, n_ent, De, devices=list(range(self.world)))
        # replicated relation table: identical init on every rank
        gr = torch.Generator(device=device).manual_seed(seed * 1000003 + 777)
        self.rel_emb = torch.empty((n_rel, Dr), dtype=torch.float32, device=device).uniform_(-hp.emb_init, hp.emb_init, generator=gr)
        self.rel_state = torch.zeros(n_rel, dtype=torch.float32, device=device)
        dist.broadcast(self.rel_emb, src=0, group=group)
        self.rel = DeviceTable.from_tensors(self.rel_emb, self.rel_state)
        # dense relation-gradient buffer [n_rel * Dr | n_rel], all-reduced as one message
        self.rbuf = torch.zeros(n_rel * Dr + n_rel, dtype=torch.float32, device=device)
        self.rg, self.rgs = self.rbuf[:n_rel * Dr], self.rbuf[n_rel * Dr:]
        _lib.check(lib.kge_set_relation_mode(self.h.raw, 1))
        # the fused step sums the relation gradients straight into the all-reduce buffer
        _lib.check(lib.kge_set_relation_buffers(self.h.raw, self.rg.data_ptr(), self.rgs.data_ptr()))
        self.eng = StepEngine(hp, self.ent, self.rel, device.index)
        self.log4 = self.eng.log4
        self._log_host = torch.zeros(4, dtype=torch.float32).pin_memory()
        dist.barrier(group=group)

    # -- one training step: forward/backward, entity Adagrad over NVLink, relation all-reduce + apply
    def step(self, node_ids, head_local=None, tail_local=None, rel_ids=None, neg_ids=None, chunk_size=None,
             neg_sample_size=None, neg_head=None, edge_weight=None, log4=None, sync_between=False, next_batch=None):
        """sync_between (tests): a cross-rank barrier between the gradient half and the update half, so that every
        rank's gradients come from the same table snapshot.
        next_batch (--async_update): the batch of the NEXT call (DeviceBatch or (node_ids, neg_ids)); its rows are
        fetched over NVLink by this step's fused kernels while they compute, so the next step starts without a gather --
        and reads rows that may lag this step's updates by one step, the staleness the reference's async update has."""
        lib, h = self.h.lib, self.h
        # gather (peer loads) .. k_chain: per-relation gradient sums land in rbuf
        # (node_ids may be a sampler.DeviceBatch: the indices then never visit the host)
        self.eng.step_begin(node_ids, head_local, tail_local, rel_ids, neg_ids, chunk_size=chunk_size,
                            neg_sample_size=neg_sample_size, neg_head=neg_head, edge_weight=edge_weight,
                            next_batch=next_batch)
        # the relation all-reduce (NCCL stream) overlaps the entity Adagrad kernel, which does not touch rbuf
        if sync_between:
            self.barrier()
        work = dist.all_reduce(self.rbuf, op=dist.ReduceOp.SUM, group=self.group, async_op=True)
        out = self.eng.step_end(log4)
        work.wait()
        _lib.check(lib.kge_rel_apply_dense(h.raw, self.rel.ref(), self.rg.data_ptr(), self.rgs.data_ptr(),
                                           float(self.hp.lr), h.stream()))
        return out

    def step_host(self, node_ids, head_local, tail_local, rel_ids, neg_ids, chunk_size, neg_sample_size, neg_head,
                  edge_weight=None, next_host=None):
        """Host index tensors.  next_host = the NEXT call's (node_ids, head_local, tail_local, rel_ids, neg_ids): they
        are uploaded now (one batch of indices crosses PCIe per step either way) and announced to the library, whose
        fused kernels then fetch that batch's rows while this step computes."""
        d = lambda t: t.to(self.device, non_blocking=True)
        up = getattr(self, "_uploaded", None)
        if up is not None and up[0] is node_ids:
            cur = up[1]
        else:
            cur = [d(node_ids), d(head_local), d(tail_local), d(rel_ids), d(neg_ids)]
        self._uploaded, nb = None, None
        if next_host is not None:
            nxt = [d(t) for t in next_host[:5]]
            self._uploaded, nb = (next_host[0], nxt), (nxt[0], nxt[4])
        out = self.step(cur[0], cur[1], cur[2], cur[3], cur[4], chunk_size, neg_sample_size, neg_head,
                        None if edge_weight is None else d(edge_weight), next_batch=nb)
        self._log_host.copy_(out, non_blocking=True)
        return self._log_host

    def evaluate(self, split, batch_size, neg_sample_size=-1, block_rows=None, seed=0):
        """Filtered ranking of this rank's slice of `split` (an evaluate.EvalSplit) over the sharded entity table.
        Returns (this rank's six sums, the sums all-reduced over the group), float64 CPU tensors; see
        evaluate.metrics_from_sums.  The evaluation runs on a handle of its own, so rows a pipelined step staged for the
        next step (kge_set_next_batch) stay staged and valid: evaluation does not write the tables."""
        from .evaluate import Evaluator
        ev = Evaluator(self.hp, self.ent, self.rel, self.device, block_rows=block_rows, seed=seed * 1000003 + self.rank)
        try:
            local = ev.run(split, batch_size, neg_sample_size).clone()
        finally:
            ev.close()
        pooled = local.clone()
        dist.all_reduce(pooled, op=dist.ReduceOp.SUM, group=self.group)
        return local.cpu(), pooled.cpu()

    def sync(self):
        torch.cuda.current_stream(self.device).synchronize()

    def close(self):
        """Unmap the local shard and the peers' (all ranks together: the memory goes when its last mapping does)."""
        if getattr(self, "_owned", None):
            self.barrier()
            self.ent_local = self.ent_state_local = None
            for ptr, nbytes in self._owned:
                _lib.check(self.h.lib.kge_shard_free(self.h.raw, ptr, nbytes))
            self._owned = []
            self.barrier()

    def barrier(self):
        """force_sync_interval analogue (train_pytorch.py:157-159): a cross-GPU barrier."""
        torch.cuda.synchronize(self.device)
        dist.barrier(group=self.group)

    def gather_entity_table(self):
        """Full [n_ent, D] table on this rank's device (for saving / evaluation)."""
        parts = [torch.empty((shard_rows(self.n_ent, self.world, r)[2] - shard_rows(self.n_ent, self.world, r)[1],
                              self.hp.entity_dim), dtype=torch.float32, device=self.device) for r in range(self.world)]
        dist.all_gather(parts, self.ent_local.contiguous(), group=self.group) if len({p.shape for p in parts}) == 1 else \
            [dist.broadcast(parts[r] if r != self.rank else self.ent_local, src=r, group=self.group) for r in range(self.world)]
        parts[self.rank] = self.ent_local
        return torch.cat(parts, 0)
