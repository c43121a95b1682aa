"""TEST INFRASTRUCTURE ONLY -- drives the UNMODIFIED reference (awslabs/dgl-ke; REFERENCE_PY below says
where a checkout is looked for) on CPU torch so that golden vectors can be generated
from the reference itself (SURVEY.md section 8c).

The reference's hot path needs DGL only for (a) a dozen `dgl.backend` tensor aliases
and (b) the sampled pos/neg graph objects.  Both are replaced here by tiny stand-ins:
the arithmetic that is recorded in tests/golden/ is executed by the reference's own
`KEModel.forward` -> `loss.backward()` -> `KEModel.update()`
(general_models.py:529-588, tensor_models.py:270-362, score_fun.py, loss.py:69-98).

This file can only run where a checkout of the reference exists.  Nothing in
the product, `-m gpu` tests, smoke() or bench.py imports it.
"""
import os
import sys
import types
import argparse

import numpy as np
import torch as th

# python/ of a checkout of the reference: KGE_REFERENCE_PY, else a `reference` directory next to this repository
REFERENCE_PY = os.path.abspath(os.environ.get("KGE_REFERENCE_PY") or os.path.join(
    os.path.dirname(os.path.abspath(__file__)), "..", "..", "reference", "python"))


def reference_available():
    return os.path.isdir(os.path.join(REFERENCE_PY, "dglke"))


def _install_stubs():
    """Register stand-in `dgl` / `ogb` modules (only what the hot path touches)."""
    if "dgl" in sys.modules and getattr(sys.modules["dgl"], "_kge_stub", False):
        return
    dgl = types.ModuleType("dgl")
    dgl._kge_stub = True
    dgl.__version__ = "0.4.3"
    be = types.ModuleType("dgl.backend")
    be.cpu = lambda: th.device("cpu")
    be.float32 = th.float32
    be.int64 = th.int64
    be.ones = lambda shape, dtype, ctx: th.ones(shape, dtype=dtype, device=ctx)
    be.zeros = lambda shape, dtype, ctx: th.zeros(shape, dtype=dtype, device=ctx)
    be.context = lambda t: t.device
    be.cat = lambda seq, dim: th.cat(seq, dim)
    be.copy_to = lambda t, ctx: t.to(ctx)
    be.asnumpy = lambda t: t.detach().cpu().numpy()
    be.sum = lambda t, dim: th.sum(t, dim)
    be.tensor = lambda data, dtype=None: th.as_tensor(data, dtype=dtype)
    be.shape = lambda t: t.shape
    be.reshape = lambda t, shape: t.reshape(shape)
    be.arange = lambda a, b: th.arange(a, b)
    be.argsort = lambda t, dim, descending: th.argsort(t, dim=dim, descending=descending)
    be.uniform = lambda shape, dtype, ctx, lo, hi: th.empty(shape, dtype=dtype, device=ctx).uniform_(lo, hi)
    be.unsqueeze = lambda t, dim: t.unsqueeze(dim)
    dgl.backend = be
    contrib = types.ModuleType("dgl.contrib")
    sampling = types.ModuleType("dgl.contrib.sampling")
    contrib.sampling = sampling
    contrib.KVClient = type("KVClient", (), {})
    contrib.KVServer = type("KVServer", (), {})
    contrib.read_ip_config = lambda *a, **k: None
    dgl.contrib = contrib
    base = types.ModuleType("dgl.base")
    base.NID, base.EID = "_ID", "_ID"
    dgl.base = base
    dep = types.ModuleType("dgl._deprecate")
    depg = types.ModuleType("dgl._deprecate.graph")
    depg.DGLGraph = type("DGLGraph", (), {})
    dep.graph = depg
    dgl._deprecate = dep
    dgl.DGLGraph = depg.DGLGraph
    ogb = types.ModuleType("ogb")
    lsc = types.ModuleType("ogb.lsc")
    lsc.WikiKG90MDataset = type("WikiKG90MDataset", (), {})
    lsc.WikiKG90MEvaluator = type("WikiKG90MEvaluator", (), {})
    ogb.lsc = lsc
    for name, mod in [("dgl", dgl), ("dgl.backend", be), ("dgl.contrib", contrib),
                      ("dgl.contrib.sampling", sampling), ("dgl.base", base),
                      ("dgl._deprecate", dep), ("dgl._deprecate.graph", depg),
                      ("ogb", ogb), ("ogb.lsc", lsc)]:
        sys.modules[name] = mod


def import_reference():
    """Return the reference's `dglke.models.general_models` module, imported unmodified."""
    if not reference_available():
        raise RuntimeError("reference tree not found at %s" % REFERENCE_PY)
    _install_stubs()
    os.environ.setdefault("DGLBACKEND", "pytorch")
    if REFERENCE_PY not in sys.path:
        sys.path.insert(0, REFERENCE_PY)
    import warnings
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        import dglke.models.general_models as gm  # noqa
    return gm


class _EdgeBatch:
    def __init__(self, src, dst, data):
        self.src, self.dst, self.data = src, dst, data


class FakePosGraph:
    """The ~8 members of the sampled positive subgraph KEModel touches (SURVEY 8b)."""

    def __init__(self, node_ids, head_local, tail_local, rel_ids, impts=None):
        self.ndata = {"id": node_ids}
        self.edata = {"id": rel_ids}
        if impts is not None:
            self.edata["impts"] = impts
        self._h, self._t = head_local, tail_local

    def all_edges(self, order="eid"):
        return self._h, self._t

    def number_of_edges(self):
        return int(self._h.shape[0])

    def apply_edges(self, fn):
        e = _EdgeBatch({"emb": self.ndata["emb"][self._h]},
                       {"emb": self.ndata["emb"][self._t]},
                       {k: v for k, v in self.edata.items()})
        self.edata.update(fn(e))


class FakeNegGraph:
    def __init__(self, neg_ids, num_chunks, chunk_size, neg_sample_size, neg_head):
        self.ndata = {"id": neg_ids}
        loc = th.arange(neg_ids.shape[0])
        self.head_nid = loc
        self.tail_nid = loc
        self.num_chunks, self.chunk_size = num_chunks, chunk_size
        self.neg_sample_size, self.neg_head = neg_sample_size, neg_head
        self.edata = {}


def make_args(**kw):
    """argparse.Namespace with the training fields KEModel / ExternalEmbedding read."""
    d = dict(gpu=[-1], mix_cpu_gpu=False, has_edge_importance=False, strict_rel_part=False,
             soft_rel_part=False, lr=0.01, regularization_coef=2e-6, regularization_norm=3,
             neg_deg_sample=False, neg_deg_sample_eval=False, loss_genre="Logsigmoid",
             neg_adversarial_sampling=False, adversarial_temperature=1.0, pairwise=False,
             margin=1.0, eval_filter=False, num_thread=1, num_proc=1, async_update=False)
    d.update(kw)
    return argparse.Namespace(**d)


def build_reference_model(model_name, n_ent, n_rel, hidden_dim, gamma, args,
                          double_ent=False, double_rel=False, seed=0):
    gm = import_reference()
    th.manual_seed(seed)
    return gm.KEModel(args, model_name, n_ent, n_rel, hidden_dim, gamma,
                      double_entity_emb=double_ent, double_relation_emb=double_rel)


def reference_step(model, node_ids, head_local, tail_local, rel_ids, neg_ids,
                   num_chunks, chunk_size, neg_sample_size, neg_head, impts=None,
                   do_update=True):
    """One reference training step (train_pytorch.py:141-152). Returns a dict of every
    intermediate the parity tests compare against."""
    pos_g = FakePosGraph(node_ids, head_local, tail_local, rel_ids, impts)
    neg_g = FakeNegGraph(neg_ids, num_chunks, chunk_size, neg_sample_size, neg_head)
    loss, log = model.forward(pos_g, neg_g, -1)
    # recompute the two score tensors exactly as forward() does, for the fixtures
    with th.no_grad():
        pos_score = pos_g.edata["score"].detach().clone()
    loss.backward()
    ent_trace = [(i.clone(), d.detach().clone(), d.grad.detach().clone()) for i, d in model.entity_emb.trace]
    rel_trace = [(i.clone(), d.detach().clone(), d.grad.detach().clone()) for i, d in model.relation_emb.trace]
    out = dict(loss=float(loss.detach()), log=dict(log), pos_score=pos_score,
               ent_trace=ent_trace, rel_trace=rel_trace)
    if do_update:
        model.update(-1)
        out["entity_emb"] = model.entity_emb.emb.detach().clone()
        out["entity_state"] = model.entity_emb.state_sum.detach().clone()
        out["relation_emb"] = model.relation_emb.emb.detach().clone()
        out["relation_state"] = model.relation_emb.state_sum.detach().clone()
    else:
        model.entity_emb.trace = []
        model.relation_emb.trace = []
    return out


def reference_neg_score(model, node_ids, head_local, tail_local, rel_ids, neg_ids,
                        num_chunks, chunk_size, neg_sample_size, neg_head):
    """pos/neg score tensors of the reference without tracing (general_models.py:348-434)."""
    pos_g = FakePosGraph(node_ids, head_local, tail_local, rel_ids)
    neg_g = FakeNegGraph(neg_ids, num_chunks, chunk_size, neg_sample_size, neg_head)
    with th.no_grad():
        pos_g.ndata["emb"] = model.entity_emb(pos_g.ndata["id"], -1, False)
        pos_g.edata["emb"] = model.relation_emb(pos_g.edata["id"], -1, False)
        pos = model.predict_score(pos_g)
        neg = model.predict_neg_score(pos_g, neg_g, trace=False,
                                      neg_deg_sample=bool(getattr(model.args, "neg_deg_sample", False)))
    return pos.clone(), neg.clone()
