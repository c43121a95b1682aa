"""KEModel -- the reference's training model object (models/general_models.py:183-680) as a thin host
mirror over libkge_b200.  Same constructor signature, attributes (entity_emb, relation_emb,
score_func, loss_gen, emb_init) and methods; the train loop of the reference keeps its shape:

    loss, log = model.forward(pos_g, neg_g, gpu_id)     # kge_forward_backward: every gradient, one stream
    loss.backward()                                     # no-op: nothing left to differentiate
    model.update(gpu_id)                                # kge_update: row-sparse Adagrad

Only the six score functions of the hot path are available (TransE_l1/l2, DistMult, ComplEx, RESCAL,
RotatE); TransR / SimplE raise (SURVEY 8f-4).
"""
import torch as th

from . import _lib
from . import engine as E
from .tensor_models import ExternalEmbedding, get_device, get_dev
from .score_fun import TransEScore, DistMultScore, ComplExScore, RESCALScore, RotatEScore, _bind_dims
from .loss import LossGenerator, LazyLog, FusedLoss

EMB_INIT_EPS = 2.0


class KEModel(object):
    def __init__(self, args, model_name, n_entities, n_relations, hidden_dim, gamma,
                 double_entity_emb=False, double_relation_emb=False):
        super(KEModel, self).__init__()
        if model_name == "TransE":
            model_name = "TransE_l2"
        if model_name not in _lib.MODEL_IDS:
            raise NotImplementedError("model %s is not on the accelerated hot path" % model_name)
        self.args = args
        self.has_edge_importance = getattr(args, "has_edge_importance", False)
        self.n_entities, self.n_relations = n_entities, n_relations
        self.model_name, self.hidden_dim = model_name, hidden_dim
        self.eps = EMB_INIT_EPS
        self.emb_init = (gamma + self.eps) / hidden_dim
        self.hyper = E.Hyper(model=model_name, hidden_dim=hidden_dim, gamma=gamma, lr=args.lr,
                             reg_coef=getattr(args, "regularization_coef", 0.0),
                             reg_norm=getattr(args, "regularization_norm", 3),
                             adversarial=getattr(args, "neg_adversarial_sampling", False),
                             adv_temperature=getattr(args, "adversarial_temperature", 1.0),
                             double_ent=double_entity_emb, double_rel=double_relation_emb,
                             loss_genre=getattr(args, "loss_genre", "Logsigmoid"), margin=getattr(args, "margin", 1.0),
                             pairwise=getattr(args, "pairwise", False),
                             neg_deg_sample=getattr(args, "neg_deg_sample", False))
        entity_dim, rel_dim = self.hyper.entity_dim, self.hyper.relation_dim
        self.entity_dim, self.rel_dim = entity_dim, rel_dim
        self.strict_rel_part = getattr(args, "strict_rel_part", False)
        self.soft_rel_part = getattr(args, "soft_rel_part", False)
        if self.strict_rel_part or self.soft_rel_part:
            raise NotImplementedError("relation partitioning (--rel_part) is replaced by the replicated relation "
                                      "table + NCCL all-reduce of dglke_b200.dist")
        device = get_device(args)
        if device.type != "cuda":
            raise _lib.KgeError("KEModel needs --gpu >= 0: the library has no CPU path")
        self.device = device
        self.loss_gen = LossGenerator(args, getattr(args, "loss_genre", "Logsigmoid"),
                                      getattr(args, "neg_adversarial_sampling", False),
                                      getattr(args, "adversarial_temperature", 1.0), getattr(args, "pairwise", False))
        self.entity_emb = ExternalEmbedding(args, n_entities, entity_dim, device)
        self.relation_emb = ExternalEmbedding(args, n_relations, rel_dim, device)
        if model_name in ("TransE_l1", "TransE_l2"):
            self.score_func = TransEScore(gamma, "l1" if model_name == "TransE_l1" else "l2")
        elif model_name == "DistMult":
            self.score_func = DistMultScore()
        elif model_name == "ComplEx":
            self.score_func = ComplExScore()
        elif model_name == "RESCAL":
            self.score_func = RESCALScore(self.hyper.relation_dim // entity_dim, entity_dim)
        elif model_name == "RotatE":
            self.score_func = RotatEScore(gamma, self.emb_init)
        _bind_dims(self.score_func, self.hyper)
        self.head_neg_score = self.score_func.create_neg(True)
        self.tail_neg_score = self.score_func.create_neg(False)
        self.head_neg_prepare = self.score_func.create_neg_prepare(True)
        self.tail_neg_prepare = self.score_func.create_neg_prepare(False)
        self._engine = None
        self.reset_parameters()

    # -- parameters -------------------------------------------------------------------------------
    def share_memory(self):
        self.entity_emb.share_memory()
        self.relation_emb.share_memory()

    def save_emb(self, path, dataset):
        self.entity_emb.save(path, dataset + "_" + self.model_name + "_entity")
        self.relation_emb.save(path, dataset + "_" + self.model_name + "_relation")
        self.score_func.save(path, dataset + "_" + self.model_name)

    def load_emb(self, path, dataset):
        self.entity_emb.load(path, dataset + "_" + self.model_name + "_entity")
        self.relation_emb.load(path, dataset + "_" + self.model_name + "_relation")
        self.score_func.load(path, dataset + "_" + self.model_name)
        self._engine = None

    def reset_parameters(self):
        self.entity_emb.init(self.emb_init)
        self.score_func.reset_parameters()
        self.relation_emb.init(self.emb_init)

    def engine(self):
        if self._engine is None or self._engine.ent is not self.entity_emb.table() \
                or self._engine.rel is not self.relation_emb.table():
            self._engine = E.StepEngine(self.hyper, self.entity_emb.table(), self.relation_emb.table(),
                                        self.device.index)
        self.hyper.lr = self.args.lr
        return self._engine

    # -- stand-alone scoring (evaluation / inference / parity tests) ---------------------------------
    def predict_score(self, g):
        self.score_func(g)
        return g.edata["score"]

    def predict_neg_score(self, pos_g, neg_g, to_device=None, gpu_id=-1, trace=False, neg_deg_sample=False):
        """Forward-only negative scores [C, Cs, Ns] (general_models.py:348-434).  neg_deg_sample (the --neg_deg_sample_eval
        case: training steps carry the flag in the step configuration instead): the chunk's own corrupted-side rows are scored
        as chunk_size extra negatives in front of the sampled ones, the score of a positive against its own row is
        multiplied by 0, and neg_g.neg_sample_size becomes chunk_size + neg_sample_size (:396-403, :417-424, :429-432)."""
        num_chunks, chunk_size, neg_sample_size = neg_g.num_chunks, neg_g.chunk_size, neg_g.neg_sample_size
        head_ids, tail_ids = pos_g.all_edges(order="eid")
        rel = pos_g.edata["emb"]

        def with_own(own_rows, neg_rows):
            own = own_rows.reshape(num_chunks, chunk_size, -1)
            cat = th.cat([own, neg_rows.reshape(num_chunks, neg_sample_size, -1)], 1)
            return cat.reshape(num_chunks * (chunk_size + neg_sample_size), -1).contiguous()

        if neg_g.neg_head:
            neg_head = self.entity_emb(neg_g.ndata["id"][neg_g.head_nid], gpu_id, trace)
            tail = pos_g.ndata["emb"][tail_ids.to(rel.device)]
            if neg_deg_sample:
                neg_head = with_own(pos_g.ndata["emb"][head_ids.to(rel.device)], neg_head)
                neg_sample_size = chunk_size + neg_sample_size
            neg_head, tail = self.head_neg_prepare(pos_g.edata["id"], num_chunks, neg_head, tail, gpu_id, trace)
            score = self.head_neg_score(neg_head, rel, tail, num_chunks, chunk_size, neg_sample_size)
        else:
            neg_tail = self.entity_emb(neg_g.ndata["id"][neg_g.tail_nid], gpu_id, trace)
            head = pos_g.ndata["emb"][head_ids.to(rel.device)]
            if neg_deg_sample:
                neg_tail = with_own(pos_g.ndata["emb"][tail_ids.to(rel.device)], neg_tail)
                neg_sample_size = chunk_size + neg_sample_size
            head, neg_tail = self.tail_neg_prepare(pos_g.edata["id"], num_chunks, head, neg_tail, gpu_id, trace)
            score = self.tail_neg_score(head, rel, neg_tail, num_chunks, chunk_size, neg_sample_size)
        if neg_deg_sample:
            neg_g.neg_sample_size = neg_sample_size
            mask = th.ones((num_chunks, chunk_size * neg_sample_size), dtype=score.dtype, device=score.device)
            mask[:, 0::(neg_sample_size + 1)] = 0
            return score * mask.reshape(num_chunks, chunk_size, neg_sample_size)
        return score

    def forward_test(self, pos_g, neg_g, logs, gpu_id=-1):
        """Ranking of each positive among its negatives (general_models.py:436-485):
        rank = 1 + #{neg >= pos}, optionally filtered by neg_g.edata['bias'] != -1."""
        pos_g.ndata["emb"] = self.entity_emb(pos_g.ndata["id"], gpu_id, False)
        pos_g.edata["emb"] = self.relation_emb(pos_g.edata["id"], gpu_id, False)
        batch_size = pos_g.number_of_edges()
        pos_scores = self.predict_score(pos_g).view(batch_size, -1)
        neg_scores = self.predict_neg_score(pos_g, neg_g, gpu_id=gpu_id, trace=False,
                                            neg_deg_sample=getattr(self.args, "neg_deg_sample_eval", False)).reshape(batch_size, -1)
        hit = neg_scores >= pos_scores
        if getattr(self.args, "eval_filter", False) and "bias" in neg_g.edata:
            hit = hit & (neg_g.edata["bias"].to(hit.device).reshape(batch_size, -1) != -1)
        ranking = (hit.sum(dim=1) + 1).cpu().tolist()
        for r in ranking:
            logs.append({"MRR": 1.0 / r, "MR": float(r), "HITS@1": 1.0 if r <= 1 else 0.0,
                         "HITS@3": 1.0 if r <= 3 else 0.0, "HITS@10": 1.0 if r <= 10 else 0.0})

    # -- the training hot path ----------------------------------------------------------------------
    def forward(self, pos_g, neg_g, gpu_id=-1):
        """gather -> positive + chunked negative scores -> loss -> every gradient, in one stream-ordered
        sequence of CUDA kernels (kge_forward_backward).  Returns (loss, log) like the reference.

        A batch that comes from the device sampler (pos_g.device_batch, dglke_b200.sampler) takes the fused
        schedule: forward = kge_step_fused_begin, update = kge_step_fused_end, 5 kernels per step; the log scalars are
        produced by the update kernel and read lazily."""
        # --neg_deg_sample (general_models.py:396-403,417-424) travels in the step configuration (Hyper.neg_deg_sample):
        # the library scores the chunk's own corrupted-side rows as extra negatives (kge_negdeg.cu)
        batch = getattr(pos_g, "device_batch", None)
        if batch is not None and not self.has_edge_importance:
            eng = self.engine()
            eng.step_begin(batch, chunk_size=neg_g.chunk_size, neg_sample_size=neg_g.neg_sample_size)
            self._fused_pending = True
            with_reg = self.hyper.reg_coef > 0.0 and self.hyper.reg_norm > 0
            return FusedLoss(eng.log4, with_reg, lazy=True), LazyLog(eng.log4, has_reg=with_reg, lazy=True, only_loss=self.hyper.pairwise)
        dev = self.device
        mv = lambda t: t if t.device == dev else t.to(dev, non_blocking=True)
        head_local, tail_local = pos_g.all_edges(order="eid")
        neg_ids = neg_g.ndata["id"][neg_g.head_nid if neg_g.neg_head else neg_g.tail_nid]
        w = mv(pos_g.edata["impts"]).float().contiguous() if self.has_edge_importance else None
        eng = self.engine()
        log4 = eng.forward_backward(mv(pos_g.ndata["id"]), mv(head_local), mv(tail_local), mv(pos_g.edata["id"]),
                                    mv(neg_ids), neg_g.chunk_size, neg_g.neg_sample_size, bool(neg_g.neg_head), w)
        with_reg = self.hyper.reg_coef > 0.0 and self.hyper.reg_norm > 0
        return FusedLoss(log4, with_reg), LazyLog(log4, has_reg=with_reg, only_loss=self.hyper.pairwise)

    def update(self, gpu_id=-1):
        if getattr(self, "_fused_pending", False):
            self.engine().step_end()
            self._fused_pending = False
        else:
            self.engine().update()
        self.score_func.update(gpu_id)

    # -- reference API kept for train loops written against it -----------------------------------------
    def create_async_update(self):
        self.entity_emb.create_async_update()

    def finish_async_update(self):
        self.entity_emb.finish_async_update()

    def prepare_relation(self, device=None):
        raise NotImplementedError("relation partitioning is not used by this multi-GPU path")

    def writeback_relation(self, rank=0, rel_parts=None):
        raise NotImplementedError("relation partitioning is not used by this multi-GPU path")

    def load_relation(self, device=None):
        raise NotImplementedError("relation partitioning is not used by this multi-GPU path")
