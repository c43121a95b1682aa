"""wgmma engine (engine=1: TMA + wgmma 3xTF32 + register epilogues) against the CPU oracle, same
tolerances as the fp32 tile engine -- the 3xTF32 split keeps fp32-level accuracy."""
import numpy as np
import pytest
import torch as th

import kge_oracle as ko
from test_gpu_parity import _random_step, _run_and_check

pytestmark = pytest.mark.gpu

SHAPES = [  # (model, hidden, gamma, n_ent, n_rel, B, Cs, Ns)
    ("DistMult", 64, 12.0, 3000, 20, 128, 128, 64),
    ("DistMult", 400, 143.0, 5000, 100, 600, 200, 200),
    ("TransE_l2", 400, 19.9, 14951, 1345, 1000, 200, 200),
    ("ComplEx", 400, 143.0, 5000, 100, 400, 200, 200),
    ("TransE_l2", 96, 10.0, 977, 13, 320, 160, 72),          # ragged: Cs != Ns, small D
    ("DistMult", 512, 143.0, 20000, 50, 512, 256, 512),      # Ns > 256: two N tiles in GEMM1
    ("DistMult", 512, 143.0, 50000, 100, 2048, 1024, 1024),  # BASELINE configs[4] chunk shape: d=512, neg=1024
]


@pytest.fixture
def umma_engine():
    from dglke_b200 import _lib
    h = _lib.get_handle(0)
    h.set_engine(1)
    yield h
    h.set_engine(-1)


@pytest.mark.parametrize("cfg", SHAPES, ids=lambda c: "%s_d%d_B%d_%dx%d" % (c[0], c[1], c[5], c[6], c[7]))
@pytest.mark.parametrize("neg_head", [False, True])
def test_umma_step_matches_oracle(umma_engine, cfg, neg_head):
    model, hidden, gamma, n_ent, n_rel, B, Cs, Ns = cfg
    hp = ko.Hyper(model=model, hidden_dim=hidden, gamma=gamma, lr=0.1, reg_coef=1e-6, reg_norm=3, adversarial=True)
    ent, es, rel, rs = ko.init_tables(hp, n_ent, n_rel, seed=3)
    es.uniform_(0.0, 1e-3)
    rs.uniform_(0.0, 1e-3)
    si, C = _random_step(hp, n_ent, n_rel, B, Cs, Ns, neg_head, seed=21)
    o = [x.clone() for x in (ent, es, rel, rs)]
    fb = ko.train_step(hp, o[0], o[1], o[2], o[3], si["node_ids"], si["head_local"], si["tail_local"], si["rel_ids"],
                       si["neg_ids"], C, Cs, Ns, neg_head)
    ref = dict(pos_score=fb["pos_score"].numpy(), neg_score=fb["neg_score"].numpy(), log=fb["log"],
               nodes_grad=fb["nodes_grad"].numpy(), negs_grad=fb["negs_grad"].numpy(), rels_grad=fb["rels_grad"].numpy(),
               ent_emb=o[0].numpy(), ent_state=o[1].numpy(), rel_emb=o[2].numpy(), rel_state=o[3].numpy())
    launches0 = umma_engine.launch_count()
    _run_and_check(hp, (ent, es, rel, rs), si, C, Cs, Ns, ref, tol=5e-5)
    assert umma_engine.launch_count() > launches0
