"""ExternalEmbedding: the reference's sparse embedding table (models/pytorch/tensor_models.py:210-407)
backed by libkge_b200.  Same constructor, attributes (`emb`, `state_sum`, `trace`) and methods; the
table lives in GPU HBM as a torch tensor, every operation on it is a CUDA kernel of the library:

  __call__  -> kge_gather   (bit-exact row gather)
  update    -> kge_adagrad  (row-sparse Adagrad over each traced (idx, grad) entry, in order)

In the fused training path KEModel.forward/update bypass the trace and call kge_forward_backward /
kge_update directly; the traced path below is what user code written against the reference's plugin
API (gather rows, compute a custom loss with autograd, call update()) keeps using.
"""
import os

import numpy as np
import torch as th

from . import engine as E

logsigmoid = th.nn.functional.logsigmoid


def get_dev(gpu):
    return th.device("cpu") if gpu < 0 else th.device("cuda:" + str(gpu))


def get_device(args):
    return th.device("cpu") if args.gpu[0] < 0 else th.device("cuda:" + str(args.gpu[0]))


def get_scalar(x):
    return x.detach().item()


def norm(x, p):
    return x.norm(p=p) ** p


def reshape(arr, x, y):
    return arr.view(x, y)


def cuda(arr, gpu):
    return arr.cuda(gpu)


def abs(val):  # noqa: A001  (name kept for interface parity)
    return th.abs(val)


def masked_select(input, mask):  # noqa: A002
    return th.masked_select(input, mask)


class ExternalEmbedding:
    def __init__(self, args, num, dim, device):
        device = th.device(device)
        if device.type != "cuda":
            # --mix_cpu_gpu's host-resident table is replaced by HBM-resident (optionally sharded) tables
            device = th.device("cuda", th.cuda.current_device()) if th.cuda.is_available() else device
        if device.type != "cuda":
            raise E._lib.KgeError("ExternalEmbedding needs a CUDA device: the library has no CPU path")
        self.gpu = getattr(args, "gpu", [device.index])
        self.args = args
        self.num, self.dim = num, dim
        self.trace = []
        self.emb = th.empty(num, dim, dtype=th.float32, device=device)
        self.state_sum = th.zeros(num, dtype=th.float32, device=device)
        self.state_step = 0
        self.has_cross_rel = False
        self.async_q = None
        self._table = None

    # -- C-ABI view -------------------------------------------------------------------------------
    def table(self):
        if self._table is None or self._table.emb_shards[0].data_ptr() != self.emb.data_ptr():
            self._table = E.DeviceTable.from_tensors(self.emb, self.state_sum)
        return self._table

    def init(self, emb_init):
        self.emb.uniform_(-emb_init, emb_init)
        self.state_sum.zero_()

    def share_memory(self):
        """The reference shares CPU tables between forked workers; HBM tables are shared between
        GPU processes through CUDA IPC instead (dglke_b200.dist) -- nothing to do for one process."""
        return None

    def __call__(self, idx, gpu_id=-1, trace=True):
        idx = idx.to(self.emb.device, non_blocking=True)
        s = E.gather(self.table(), idx)
        if trace:
            data = s.requires_grad_(True)
            self.trace.append((idx, data))
            return data
        return s

    def update(self, gpu_id=-1):
        self.state_step += 1
        lr = self.args.lr
        for idx, data in self.trace:
            if data.grad is None:
                continue
            E.adagrad(self.table(), idx, data.grad.data, lr)
        self.trace = []

    def create_async_update(self):
        """--async_update overlaps the CPU-side update with GPU compute in the reference
        (tensor_models.py:136-175).  Here the update is a stream-ordered GPU kernel that already
        runs asynchronously to the host, so there is no helper process to create."""
        self.async_q = None

    def finish_async_update(self):
        return None

    def curr_emb(self):
        return th.cat([data for _, data in self.trace], 0)

    def save(self, path, name):
        np.save(os.path.join(path, name + ".npy"), self.emb.cpu().detach().numpy())

    def load(self, path, name):
        arr = th.from_numpy(np.load(os.path.join(path, name + ".npy"))).to(th.float32)
        self.emb = arr.to(self.emb.device).contiguous()
        self.num, self.dim = self.emb.shape
        if self.state_sum.shape[0] != self.num:
            self.state_sum = th.zeros(self.num, dtype=th.float32, device=self.emb.device)
        self._table = None
