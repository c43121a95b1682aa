"""TEST INFRASTRUCTURE ONLY -- CPU oracle for the KGE training hot path.

A torch-fp32 CPU restatement of the per-step arithmetic of awslabs/dgl-ke
(gather -> score over 1 positive + chunk-shared negatives -> logsigmoid /
self-adversarial loss -> autograd -> row-sparse Adagrad).  It exists so that the
parity tests, `__graft_entry__.smoke()` and `bench.py`'s `cpu_baseline` /
`--impl reference` legs have a checker that needs nothing but torch (the reference
tree itself does not).  NOTHING in the product path may import this module.

Parity is PINNED: tests/test_oracle_golden.py checks every function below against
fixtures in tests/golden/ that were produced by the *unmodified reference* driven by
oracle/ref_harness.py (generator: oracle/gen_golden.py).

Each function cites the reference lines (relative to python/dglke of awslabs/dgl-ke) it
follows.  Layout conventions (SURVEY.md Appendix A):
  * tables are fp32 row-major [num, dim]; indices int64
  * ComplEx rows are [re | im]; RotatE entity rows are [re | im], relation rows are phases
  * RESCAL relation rows are M_r row-major [rel_dim, ent_dim]
  * chunk c owns positives [c*Cs, (c+1)*Cs) and negatives [c*Ns, (c+1)*Ns)
"""
from dataclasses import dataclass
import math

import torch as th

MODELS = ("TransE_l1", "TransE_l2", "DistMult", "ComplEx", "RESCAL", "RotatE")


@dataclass
class Hyper:
    model: str = "TransE_l2"
    hidden_dim: int = 400
    gamma: float = 12.0
    lr: float = 0.01
    reg_coef: float = 2e-6
    reg_norm: int = 3
    adversarial: bool = False
    adv_temperature: float = 1.0
    double_ent: bool = False
    double_rel: bool = False
    loss_genre: str = "Logsigmoid"      # models/pytorch/loss.py:41-62
    margin: float = 1.0
    pairwise: bool = False
    neg_deg_sample: bool = False        # models/general_models.py:396-403,417-424,429-432

    @property
    def emb_init(self):
        # models/general_models.py:217-218  (gamma + 2.0) / hidden_dim
        return (self.gamma + 2.0) / self.hidden_dim

    @property
    def entity_dim(self):
        return 2 * self.hidden_dim if self.double_ent else self.hidden_dim

    @property
    def relation_dim(self):
        # models/general_models.py:219-236 ; RESCAL stores a full matrix per relation
        rd = 2 * self.hidden_dim if self.double_rel else self.hidden_dim
        return rd * self.entity_dim if self.model == "RESCAL" else rd


def canonical(model):
    return "TransE_l2" if model == "TransE" else model


# --------------------------------------------------------------------------- a3
def gather(table, idx):
    """ExternalEmbedding.__call__  (models/pytorch/tensor_models.py:292): emb[idx]."""
    return table[idx]


# --------------------------------------------------------------------------- a4
def _split(x):
    half = x.shape[-1] // 2
    return x[..., :half], x[..., half:]


def positive_score(hp, h, r, t):
    """score_func.edge_func on already-gathered rows h,t [B,De], r [B,Dr] -> [B].

    TransE score_fun.py:54-59, DistMult :229-235, ComplEx :297-307, RESCAL :387-394,
    RotatE :460-472."""
    m = canonical(hp.model)
    if m in ("TransE_l1", "TransE_l2"):
        return hp.gamma - th.norm(h + r - t, p=1 if m == "TransE_l1" else 2, dim=-1)
    if m == "DistMult":
        return th.sum(h * r * t, dim=-1)
    if m == "ComplEx":
        hr, hi = th.chunk(h, 2, dim=-1)
        tr, ti = th.chunk(t, 2, dim=-1)
        rr, ri = th.chunk(r, 2, dim=-1)
        return th.sum(hr * tr * rr + hi * ti * rr + hr * ti * ri - hi * tr * ri, -1)
    if m == "RESCAL":
        mat = r.view(-1, r.shape[-1] // h.shape[-1], h.shape[-1])
        return th.sum(h * th.matmul(mat, t.unsqueeze(-1)).squeeze(-1), dim=-1)
    if m == "RotatE":
        hr, hi = th.chunk(h, 2, dim=-1)
        tr, ti = th.chunk(t, 2, dim=-1)
        phase = r / (hp.emb_init / math.pi)
        c, s = th.cos(phase), th.sin(phase)
        dre = hr * c - hi * s - tr
        dim_ = hr * s + hi * c - ti
        return hp.gamma - th.stack([dre, dim_], dim=0).norm(dim=0).sum(-1)
    raise ValueError(m)


# --------------------------------------------------------------------------- a5
def _l2_pairs(a, b):
    """batched_l2_dist (score_fun.py:26-34): |a|^2 + |b|^2 - 2 a.b, clamp 1e-30, sqrt."""
    a2 = a.norm(dim=-1).pow(2)
    b2 = b.norm(dim=-1).pow(2)
    sq = th.baddbmm(b2.unsqueeze(-2), a, b.transpose(-2, -1), alpha=-2).add_(a2.unsqueeze(-1))
    return sq.clamp_min_(1e-30).sqrt_()


def negative_score(hp, heads, rels, tails, num_chunks, chunk_size, neg_sample_size, neg_head):
    """score_func.create_neg(neg_head)(heads, relations, tails, C, Cs, Ns) -> [C, Cs, Ns].

    neg_head=False: heads/rels are the positives' rows [C*Cs, .], tails the negative rows
    [C*Ns, De].  neg_head=True: heads are the negative rows, tails/rels the positives'.
    TransE score_fun.py:91-108, DistMult :268-286, ComplEx :345-376, RESCAL :427-449 (its
    tail branch multiplies M_r by the HEAD, i.e. scores h^T M_r^T t' -- reproduced),
    RotatE :512-554."""
    m = canonical(hp.model)
    C, Cs, Ns = num_chunks, chunk_size, neg_sample_size
    pos_e = tails if neg_head else heads        # the positive-side entity rows
    neg_e = heads if neg_head else tails        # the corrupting rows
    D = pos_e.shape[1]
    if m in ("TransE_l1", "TransE_l2"):
        a = (pos_e - rels) if neg_head else (pos_e + rels)
        a = a.reshape(C, Cs, D)
        b = neg_e.reshape(C, Ns, D)
        dist = th.cdist(a, b, p=1) if m == "TransE_l1" else _l2_pairs(a, b)
        return hp.gamma - dist
    if m == "DistMult":
        a = (pos_e * rels).reshape(C, Cs, D)
        return th.bmm(a, neg_e.reshape(C, Ns, D).transpose(1, 2))
    if m in ("ComplEx", "RotatE"):
        er, ei = pos_e[..., :D // 2], pos_e[..., D // 2:]
        if m == "ComplEx":
            rr, ri = rels[..., :D // 2], rels[..., D // 2:]
        else:
            phase = rels / (hp.emb_init / math.pi)
            rr, ri = th.cos(phase), th.sin(phase)
        if neg_head:      # conj(r) * t
            re, im = er * rr + ei * ri, -er * ri + ei * rr
        else:             # h * r
            re, im = er * rr - ei * ri, er * ri + ei * rr
        a = th.cat((re, im), dim=-1)
        if m == "ComplEx":
            return th.bmm(a.reshape(C, Cs, D), neg_e.reshape(C, Ns, D).transpose(1, 2))
        diff = a.reshape(C, Cs, 1, D) - neg_e.reshape(C, 1, Ns, D)
        mod = th.stack([diff[..., :D // 2], diff[..., D // 2:]], dim=-1).norm(dim=-1)
        return hp.gamma - mod.sum(-1)
    if m == "RESCAL":
        mat = rels.view(-1, rels.shape[-1] // D, D)
        a = th.matmul(mat, pos_e.unsqueeze(-1)).squeeze(-1).reshape(C, Cs, D)
        return th.bmm(a, neg_e.reshape(C, Ns, D).transpose(1, 2))
    raise ValueError(m)


# --------------------------------------------------------------------------- a7
def criterion(hp, score, label):
    """The four loss criteria (models/pytorch/loss.py:10-38)."""
    if hp.loss_genre == "Hinge":
        loss = hp.margin - label * score
        return th.where(loss < 0, th.zeros_like(loss), loss)          # `loss[loss < 0] = 0`
    if hp.loss_genre == "Logistic":
        return th.nn.functional.softplus(-label * score)
    if hp.loss_genre == "BCE":
        sg = th.sigmoid(score)
        return -(label * th.log(sg) + (1 - label) * th.log(1 - sg))
    if hp.loss_genre == "Logsigmoid":
        return -th.nn.functional.logsigmoid(label * score)
    raise ValueError("loss genre %s is not support" % hp.loss_genre)


def loss_terms(hp, pos_score, neg_score, edge_weight=None):
    """LossGenerator.get_total_loss (models/pytorch/loss.py:41-98).

    pos_score [B], neg_score [B, Ns].  Returns (loss tensor, log dict).  With an edge
    weight the reference views it [B,1] and multiplies the [B] positive loss by it, which
    broadcasts to [B,B] (loss.py:75,82) -- reproduced.  pairwise (loss.py:76-80): one term per
    (positive, negative) pair, plain mean, no adversarial weighting, log holds 'loss' only."""
    w = 1 if edge_weight is None else edge_weight.view(-1, 1)
    if hp.pairwise:
        if hp.loss_genre not in ("Logistic", "Hinge"):
            raise ValueError("%s loss cannot be applied to pairwise loss function" % hp.loss_genre)
        if hp.adversarial:
            raise ValueError("loss cannot be pairwise and adversarial sampled")      # base_loss.py:83-84
        loss = th.mean(criterion(hp, pos_score.unsqueeze(-1) - neg_score, 1) * w)
        return loss, {"loss": float(loss.detach())}
    neg_label = 0 if hp.loss_genre == "BCE" else -1
    pos_l = criterion(hp, pos_score, 1) * w
    neg_l = criterion(hp, neg_score, neg_label) * w
    if hp.adversarial:
        p = th.softmax(neg_score * hp.adv_temperature, dim=-1).detach()
        neg_l = th.sum(p * neg_l, dim=-1)
    else:
        neg_l = th.mean(neg_l, dim=-1)
    neg_l, pos_l = th.mean(neg_l), th.mean(pos_l)
    loss = (neg_l + pos_l) / 2
    return loss, {"pos_loss": float(pos_l.detach()), "neg_loss": float(neg_l.detach()),
                  "loss": float(loss.detach())}


# --------------------------------------------------------------------------- a10
def adagrad_entry(emb, state_sum, idx, grad, lr):
    """One trace entry of ExternalEmbedding.update (tensor_models.py:316-361), in place:
    every row's mean(g^2) is added to state_sum first (duplicates accumulate), then each
    row (duplicates included) is scaled by the FINAL state and added to emb."""
    gs = (grad * grad).mean(1)
    state_sum.index_add_(0, idx, gs)
    std = state_sum[idx].sqrt_().add_(1e-10).unsqueeze(1)
    emb.index_add_(0, idx, (-lr * grad / std))


# --------------------------------------------------------------------------- a12
def forward_backward(hp, ent_emb, rel_emb, node_ids, head_local, tail_local, rel_ids, neg_ids,
                     num_chunks, chunk_size, neg_sample_size, neg_head, edge_weight=None):
    """KEModel.forward + loss.backward() (general_models.py:529-578, train_pytorch.py:141-145).

    Returns dict(pos_score, neg_score [B,Ns], loss, log, and the three traced leaves with
    their gradients: nodes (unique positive nodes), negs, rels)."""
    nodes = gather(ent_emb, node_ids).clone().requires_grad_(True)       # trace entry 1 (entity)
    rels = gather(rel_emb, rel_ids).clone().requires_grad_(True)         # trace entry 1 (relation)
    h, t = nodes[head_local], nodes[tail_local]
    pos = positive_score(hp, h, rels, t)
    negs = gather(ent_emb, neg_ids).clone().requires_grad_(True)         # trace entry 2 (entity)
    corrupt = negs
    if hp.neg_deg_sample:
        # general_models.py:396-403 / 417-424: the chunk's own heads (head mode) / tails (tail mode) -- rows of the NODE
        # leaf, not a new traced tensor -- are put in front of the sampled negatives of every chunk, and the score of a
        # positive against its own row is multiplied by 0 (mask[:, 0::(Ns' + 1)] = 0 on the [C, Cs * Ns'] view)
        own = (h if neg_head else t).reshape(num_chunks, chunk_size, -1)
        corrupt = th.cat([own, negs.reshape(num_chunks, neg_sample_size, -1)], 1)
        neg_sample_size = chunk_size + neg_sample_size
        corrupt = corrupt.reshape(num_chunks * neg_sample_size, -1)
    if neg_head:
        neg = negative_score(hp, corrupt, rels, t, num_chunks, chunk_size, neg_sample_size, True)
    else:
        neg = negative_score(hp, h, rels, corrupt, num_chunks, chunk_size, neg_sample_size, False)
    if hp.neg_deg_sample:
        mask = th.ones(num_chunks, chunk_size * neg_sample_size, dtype=neg.dtype)
        mask[:, 0::(neg_sample_size + 1)] = 0
        neg = neg * mask.reshape(num_chunks, chunk_size, neg_sample_size)          # general_models.py:429-432
    neg = neg.reshape(-1, neg_sample_size)
    loss, log = loss_terms(hp, pos, neg, edge_weight)
    if hp.reg_coef > 0.0 and hp.reg_norm > 0:
        # general_models.py:572-576: every traced row, duplicates counted
        ent_rows = th.cat([nodes, negs], 0)
        reg = hp.reg_coef * (ent_rows.norm(p=hp.reg_norm) ** hp.reg_norm
                             + rels.norm(p=hp.reg_norm) ** hp.reg_norm)
        log["regularization"] = float(reg.detach())
        loss = loss + reg
    loss.backward()
    return dict(pos_score=pos.detach(), neg_score=neg.detach(), loss=float(loss.detach()), log=log,
                nodes=nodes.detach(), nodes_grad=nodes.grad, negs=negs.detach(), negs_grad=negs.grad,
                rels=rels.detach(), rels_grad=rels.grad)


def train_step(hp, ent_emb, ent_state, rel_emb, rel_state, node_ids, head_local, tail_local,
               rel_ids, neg_ids, num_chunks, chunk_size, neg_sample_size, neg_head,
               edge_weight=None):
    """One full step, tables updated in place (train_pytorch.py:141-152).  Update order:
    entity table entries [unique positive nodes, negatives], then relation table
    (general_models.py:586-588)."""
    fb = forward_backward(hp, ent_emb, rel_emb, node_ids, head_local, tail_local, rel_ids, neg_ids,
                          num_chunks, chunk_size, neg_sample_size, neg_head, edge_weight)
    with th.no_grad():
        adagrad_entry(ent_emb, ent_state, node_ids, fb["nodes_grad"], hp.lr)
        adagrad_entry(ent_emb, ent_state, neg_ids, fb["negs_grad"], hp.lr)
        adagrad_entry(rel_emb, rel_state, rel_ids, fb["rels_grad"], hp.lr)
    return fb


def init_tables(hp, n_ent, n_rel, seed=0):
    """ExternalEmbedding.init (tensor_models.py:240-249): U(-emb_init, emb_init), zero state.
    The entity table is drawn first, then the relation table (general_models.py:322-330)."""
    g = th.Generator().manual_seed(seed)
    e = hp.emb_init
    ent = th.empty(n_ent, hp.entity_dim).uniform_(-e, e, generator=g)
    rel = th.empty(n_rel, hp.relation_dim).uniform_(-e, e, generator=g)
    return ent, th.zeros(n_ent), rel, th.zeros(n_rel)


def rank_of_positive(pos_score, neg_score):
    """KEModel.forward_test ranking (general_models.py:473-485, unfiltered):
    rank_i = 1 + #{j : neg_ij >= pos_i}."""
    return 1 + (neg_score >= pos_score.view(-1, 1)).sum(dim=1)
