"""Generates tests/golden/*.npz from the UNMODIFIED reference (KGE_REFERENCE_PY names its
python/ directory):   python oracle/gen_golden.py

Every array in a fixture is an output of the reference's own code path
(KEModel.forward -> loss.backward() -> KEModel.update, predict_neg_score) driven through
oracle/ref_harness.py; the inputs are seeded numpy draws.  TEST INFRASTRUCTURE ONLY.
"""
import os
import sys
import json

import numpy as np
import torch as th

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import ref_harness as rh  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")

# (case name, model, dict of overrides)
CASES = []
for model in ("TransE_l1", "TransE_l2", "DistMult", "ComplEx", "RESCAL", "RotatE"):
    for adv in (False, True):
        CASES.append(("%s_%s" % (model, "adv" if adv else "uni"), model, dict(adv=adv)))
# ragged shapes: chunk_size != neg_sample_size, and one chunk only
CASES.append(("TransE_l2_cs6_ns4", "TransE_l2", dict(adv=True, chunk=6, neg=4, batch=12)))
CASES.append(("DistMult_cs2_ns8", "DistMult", dict(adv=False, chunk=2, neg=8, batch=8)))
CASES.append(("ComplEx_onechunk", "ComplEx", dict(adv=True, chunk=8, neg=8, batch=8)))
# heavy duplication: 6 entities only
CASES.append(("TransE_l2_dups", "TransE_l2", dict(adv=True, n_ent=6, n_rel=2)))
# edge importance weights (loss.py:75,82 broadcasting quirk)
CASES.append(("TransE_l2_impts", "TransE_l2", dict(adv=True, impts=True)))
# regularisation off / L2 regulariser
CASES.append(("DistMult_noreg", "DistMult", dict(adv=False, reg_coef=0.0)))
CASES.append(("ComplEx_reg2", "ComplEx", dict(adv=True, reg_norm=2, reg_coef=1e-3)))
# tensor-core shapes (D >= 32, chunk / neg multiples of 8): the tensor-core kernels are pinned against the reference directly
CASES.append(("tc_TransE_l2_adv", "TransE_l2", dict(adv=True, hidden=32, batch=16, chunk=8, neg=8, n_ent=60)))
CASES.append(("tc_TransE_l2_ragged_impts", "TransE_l2", dict(adv=True, hidden=40, batch=32, chunk=16, neg=8, n_ent=60, impts=True)))
CASES.append(("tc_DistMult_uni", "DistMult", dict(adv=False, hidden=32, batch=16, chunk=8, neg=16, n_ent=60)))
CASES.append(("tc_ComplEx_adv", "ComplEx", dict(adv=True, hidden=32, batch=16, chunk=8, neg=8, n_ent=60)))
CASES.append(("tc_RESCAL_adv", "RESCAL", dict(adv=True, hidden=32, batch=16, chunk=8, neg=8, n_ent=60, n_rel=3)))


# the other loss criteria and the pairwise form (loss.py:10-62,76-80)
CASES.append(("loss_Hinge_TransE_l2_adv", "TransE_l2", dict(adv=True, loss_genre="Hinge", margin=1.0, gamma=4.0)))
CASES.append(("loss_Hinge_DistMult_uni_impts", "DistMult", dict(adv=False, loss_genre="Hinge", margin=0.5, impts=True)))
CASES.append(("loss_Logistic_ComplEx_adv", "ComplEx", dict(adv=True, loss_genre="Logistic")))
CASES.append(("loss_BCE_TransE_l1_uni", "TransE_l1", dict(adv=False, loss_genre="BCE")))
CASES.append(("loss_pw_Logistic_DistMult", "DistMult", dict(adv=False, loss_genre="Logistic", pairwise=True)))
CASES.append(("loss_pw_Hinge_TransE_l2_impts", "TransE_l2", dict(adv=False, loss_genre="Hinge", margin=2.0, pairwise=True,
                                                                   impts=True, gamma=4.0)))
CASES.append(("tc_loss_pw_Hinge_RotatE", "RotatE", dict(adv=False, loss_genre="Hinge", margin=1.0, pairwise=True, hidden=16,
                                                        batch=16, chunk=8, neg=8, n_ent=60)))
CASES.append(("tc_loss_Hinge_ComplEx", "ComplEx", dict(adv=True, loss_genre="Hinge", margin=1.0, hidden=32, batch=16,
                                                       chunk=8, neg=8, n_ent=60)))


# --neg_deg_sample (general_models.py:396-403,417-424,429-432): the chunk's own corrupted-side rows as extra negatives
for _m in ("TransE_l1", "TransE_l2", "DistMult", "ComplEx", "RESCAL", "RotatE"):
    CASES.append(("negdeg_%s" % _m, _m, dict(adv=(_m != "DistMult"), neg_deg=True, n_ent=30)))
CASES.append(("negdeg_TransE_l2_ragged_impts", "TransE_l2", dict(adv=True, neg_deg=True, chunk=6, neg=4, batch=12, impts=True)))
CASES.append(("tc_negdeg_ComplEx", "ComplEx", dict(adv=True, neg_deg=True, hidden=32, batch=16, chunk=8, neg=8, n_ent=60)))
CASES.append(("tc_negdeg_TransE_l2_hinge", "TransE_l2", dict(adv=False, neg_deg=True, hidden=32, batch=16, chunk=8, neg=16, n_ent=60,
                                                            loss_genre="Hinge", margin=2.0, gamma=4.0)))


def one_case(name, model, o):
    n_ent, n_rel = o.get("n_ent", 40), o.get("n_rel", 5)
    hidden = o.get("hidden", 8)
    gamma = o.get("gamma", 12.0 if model not in ("TransE_l2",) else 19.9)
    batch, chunk, neg = o.get("batch", 12), o.get("chunk", 4), o.get("neg", 4)
    double_ent = model == "RotatE"
    args = rh.make_args(lr=o.get("lr", 0.25), regularization_coef=o.get("reg_coef", 2e-4),
                        regularization_norm=o.get("reg_norm", 3),
                        neg_adversarial_sampling=o["adv"], adversarial_temperature=o.get("temp", 1.5),
                        has_edge_importance=bool(o.get("impts", False)),
                        loss_genre=o.get("loss_genre", "Logsigmoid"), margin=o.get("margin", 1.0),
                        pairwise=bool(o.get("pairwise", False)), neg_deg_sample=bool(o.get("neg_deg", False)))
    m = rh.build_reference_model(model, n_ent, n_rel, hidden, gamma, args, double_ent=double_ent, seed=7)
    rng = np.random.default_rng(1234)
    fx = dict(ent_emb0=m.entity_emb.emb.clone().numpy(), rel_emb0=m.relation_emb.emb.clone().numpy())
    meta = dict(model=model, n_ent=n_ent, n_rel=n_rel, hidden_dim=hidden, gamma=gamma, lr=args.lr,
                reg_coef=args.regularization_coef, reg_norm=args.regularization_norm,
                adversarial=bool(o["adv"]), adv_temperature=args.adversarial_temperature,
                double_ent=double_ent, double_rel=False, batch=batch, chunk_size=chunk,
                neg_sample_size=neg, num_chunks=batch // chunk, steps=2,
                has_edge_importance=bool(o.get("impts", False)),
                loss_genre=o.get("loss_genre", "Logsigmoid"), margin=o.get("margin", 1.0),
                pairwise=bool(o.get("pairwise", False)), neg_deg_sample=bool(o.get("neg_deg", False)))
    C = batch // chunk
    for step in range(2):
        neg_head = (step % 2 == 1)          # sampler.py:853-859: tail first, then head
        h = rng.integers(0, n_ent, batch)
        t = rng.integers(0, n_ent, batch)
        r = rng.integers(0, n_rel, batch)
        ng = rng.integers(0, n_ent, C * neg)
        nodes, inv = np.unique(np.concatenate([h, t]), return_inverse=True)
        hl, tl = inv[:batch], inv[batch:]
        w = rng.uniform(0.5, 1.5, batch).astype(np.float32) if o.get("impts") else None
        T = lambda a: th.from_numpy(np.ascontiguousarray(a))
        pos, negs = rh.reference_neg_score(m, T(nodes), T(hl), T(tl), T(r), T(ng), C, chunk, neg, neg_head)
        out = rh.reference_step(m, T(nodes), T(hl), T(tl), T(r), T(ng), C, chunk, neg, neg_head,
                                impts=None if w is None else T(w))
        p = "s%d_" % step
        fx[p + "node_ids"], fx[p + "head_local"], fx[p + "tail_local"] = nodes, hl, tl
        fx[p + "rel_ids"], fx[p + "neg_ids"] = r, ng
        fx[p + "neg_head"] = np.array(int(neg_head))
        if w is not None:
            fx[p + "edge_weight"] = w
        fx[p + "pos_score"] = pos.numpy()
        fx[p + "neg_score"] = negs.numpy().reshape(batch, -1)           # [B, Ns] or, with neg_deg_sample, [B, Cs + Ns]
        assert np.array_equal(pos.numpy(), out["pos_score"].numpy())
        fx[p + "loss"] = np.array(out["loss"], dtype=np.float64)
        for k in ("pos_loss", "neg_loss", "loss", "regularization"):
            fx[p + "log_" + k] = np.array(out["log"].get(k, 0.0), dtype=np.float64)
        (i0, d0, g0), (i1, d1, g1) = out["ent_trace"]
        assert np.array_equal(i0.numpy(), nodes) and np.array_equal(i1.numpy(), ng)
        fx[p + "nodes"], fx[p + "nodes_grad"] = d0.numpy(), g0.numpy()
        fx[p + "negs"], fx[p + "negs_grad"] = d1.numpy(), g1.numpy()
        (ir, dr, gr), = out["rel_trace"]
        fx[p + "rels"], fx[p + "rels_grad"] = dr.numpy(), gr.numpy()
        fx[p + "ent_emb"], fx[p + "ent_state"] = out["entity_emb"].numpy(), out["entity_state"].numpy()
        fx[p + "rel_emb"], fx[p + "rel_state"] = out["relation_emb"].numpy(), out["relation_state"].numpy()
    fx["meta"] = np.array(json.dumps(meta))
    np.savez_compressed(os.path.join(OUT, name + ".npz"), **fx)
    return meta


if __name__ == "__main__":
    os.makedirs(OUT, exist_ok=True)
    only = sys.argv[1:]                  # optional: generate just the named cases / prefixes
    for name, model, o in CASES:
        if only and not any(name.startswith(x) for x in only):
            continue
        meta = one_case(name, model, o)
        print("wrote", name, meta["model"], "B", meta["batch"], "Cs", meta["chunk_size"], "Ns", meta["neg_sample_size"])
