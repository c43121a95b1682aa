"""Pins oracle/kge_oracle.py (the CPU restatement the GPU tests compare against) against the
golden vectors produced by the unmodified reference (oracle/gen_golden.py).  CPU only."""
import numpy as np
import pytest
import torch as th

import kge_oracle as ko
from golden_util import golden_cases, load_case, hyper_from_meta, step_inputs, tables_before

# same torch ops in the same order as the reference: observed bit-identical on the generating
# machine; 2e-6 absorbs a different BLAS on another host.
TOL = dict(rtol=2e-6, atol=2e-6)


@pytest.mark.parametrize("name", golden_cases())
def test_oracle_matches_reference_golden(name):
    meta, z = load_case(name)
    hp = hyper_from_meta(meta)
    C, Cs, Ns = meta["num_chunks"], meta["chunk_size"], meta["neg_sample_size"]
    for step in range(meta["steps"]):
        p = "s%d_" % step
        si = step_inputs(z, step)
        ent, ent_s, rel, rel_s = tables_before(z, step)     # each step starts from the reference's tables
        fb = ko.train_step(hp, ent, ent_s, rel, rel_s, si["node_ids"], si["head_local"], si["tail_local"],
                           si["rel_ids"], si["neg_ids"], C, Cs, Ns, si["neg_head"], si["edge_weight"])
        np.testing.assert_array_equal(fb["nodes"].numpy(), z[p + "nodes"])        # gather: bit exact
        np.testing.assert_array_equal(fb["negs"].numpy(), z[p + "negs"])
        np.testing.assert_array_equal(fb["rels"].numpy(), z[p + "rels"])
        np.testing.assert_allclose(fb["pos_score"].numpy(), z[p + "pos_score"], **TOL)
        np.testing.assert_allclose(fb["neg_score"].numpy(), z[p + "neg_score"], **TOL)
        for k in ("pos_loss", "neg_loss", "loss", "regularization"):
            if k in fb["log"]:
                np.testing.assert_allclose(fb["log"][k], float(z[p + "log_" + k]), rtol=1e-6, atol=1e-9)
        np.testing.assert_allclose(fb["loss"], float(z[p + "loss"]), rtol=1e-6)
        for k in ("nodes_grad", "negs_grad", "rels_grad"):
            np.testing.assert_allclose(fb[k].numpy(), z[p + k], rtol=2e-5, atol=1e-8)
        np.testing.assert_allclose(ent.numpy(), z[p + "ent_emb"], rtol=1e-5, atol=1e-7)
        np.testing.assert_allclose(ent_s.numpy(), z[p + "ent_state"], rtol=1e-5, atol=1e-12)
        np.testing.assert_allclose(rel.numpy(), z[p + "rel_emb"], rtol=1e-5, atol=1e-7)
        np.testing.assert_allclose(rel_s.numpy(), z[p + "rel_state"], rtol=1e-5, atol=1e-12)


def test_init_tables_range():
    hp = ko.Hyper(model="RotatE", hidden_dim=8, gamma=12.0, double_ent=True)
    ent, es, rel, rs = ko.init_tables(hp, 10, 3)
    assert ent.shape == (10, 16) and rel.shape == (3, 8)
    assert float(ent.abs().max()) <= hp.emb_init and float(es.sum()) == 0.0


def test_rank_of_positive():
    pos = th.tensor([1.0, 0.0])
    neg = th.tensor([[2.0, 1.0, 0.5], [-1.0, -2.0, -3.0]])
    assert ko.rank_of_positive(pos, neg).tolist() == [3, 1]
