"""k_prep's row blocks against the CPU oracle.  k_prep runs one CTA per (chunk, 32-row block) and writes the transposed
operand slabs from a shared-memory copy of the block, so the shapes here are the ones where the block geometry changes:
a single partial block (8 rows), exact blocks (32), the fused kernel's widest chunk (240 = 7 full blocks + 16 rows),
a partial block on one side only, D = 32 (one column block), D = 40 (ComplEx with its re/im boundary inside the first
column block), D = 520 (more than 48 KB of staging) and the staging limit, d = 1792 / 1800.  Full step, same tolerances
as the other wgmma-engine tests."""
import pytest

import kge_oracle as ko
from test_gpu_parity import _random_step, _run_and_check

pytestmark = pytest.mark.gpu

SHAPES = [  # (model, hidden, gamma, n_ent, n_rel, B, Cs, Ns)
    ("TransE_l2", 32, 10.0, 500, 7, 64, 8, 8),              # one partial block per chunk on both sides
    ("DistMult", 32, 12.0, 800, 9, 128, 32, 8),             # exact edge blocks, partial negative blocks
    ("TransE_l2", 40, 10.0, 977, 13, 240, 40, 32),          # partial edge blocks, exact negative blocks
    ("ComplEx", 40, 12.0, 1000, 11, 96, 32, 40),            # re/im boundary at column 20
    ("TransE_l2", 400, 19.9, 5000, 100, 480, 240, 240),     # fused maximum: 8 blocks, the last with 16 rows
    ("DistMult", 520, 143.0, 3000, 20, 160, 32, 32),        # staging beyond 48 KB: the kernel opts in
    ("ComplEx", 520, 143.0, 3000, 20, 240, 240, 8),
]


def _check(model, hidden, gamma, n_ent, n_rel, B, Cs, Ns, neg_head, adversarial=True):
    hp = ko.Hyper(model=model, hidden_dim=hidden, gamma=gamma, lr=0.1, reg_coef=1e-6, reg_norm=3, adversarial=adversarial)
    ent, es, rel, rs = ko.init_tables(hp, n_ent, n_rel, seed=3)
    es.uniform_(0.0, 1e-3)
    rs.uniform_(0.0, 1e-3)
    si, C = _random_step(hp, n_ent, n_rel, B, Cs, Ns, neg_head, seed=41)
    o = [x.clone() for x in (ent, es, rel, rs)]
    fb = ko.train_step(hp, o[0], o[1], o[2], o[3], si["node_ids"], si["head_local"], si["tail_local"], si["rel_ids"],
                       si["neg_ids"], C, Cs, Ns, neg_head)
    ref = dict(pos_score=fb["pos_score"].numpy(), neg_score=fb["neg_score"].numpy(), log=fb["log"],
               nodes_grad=fb["nodes_grad"].numpy(), negs_grad=fb["negs_grad"].numpy(), rels_grad=fb["rels_grad"].numpy(),
               ent_emb=o[0].numpy(), ent_state=o[1].numpy(), rel_emb=o[2].numpy(), rel_state=o[3].numpy())
    _run_and_check(hp, (ent, es, rel, rs), si, C, Cs, Ns, ref, tol=5e-5)


@pytest.mark.parametrize("cfg", SHAPES, ids=lambda c: "%s_d%d_B%d_%dx%d" % (c[0], c[1], c[5], c[6], c[7]))
@pytest.mark.parametrize("neg_head", [False, True])
def test_prep_row_blocks_match_oracle(cfg, neg_head):
    _check(*cfg, neg_head)


@pytest.mark.parametrize("hidden,wgmma", [(1792, True), (1800, False)])
def test_prep_staging_limit(hidden, wgmma):
    """d = 1792 is the widest row whose 32-row block fits the 227 KB of shared memory a CTA may have (225 KB): it runs on
    the wgmma engine.  d = 1800 would need 228.5 KB and runs on the fp32 tiles, which need no transposed slabs.  Both
    against the oracle; the kernel names of the step say which engine ran.  TransE_l2: its scores are gamma - distance,
    so the score tolerance is relative to gamma.  A bilinear score summed over 1792 products on the tensor cores carries
    more rounding than the test's 2e-6 of the largest score (the engine's limit at this depth, not k_prep's)."""
    from dglke_b200 import _lib
    h = _lib.get_handle(0)
    h.profile_enable(True)
    try:
        _check("TransE_l2", hidden, 19.9, 2000, 10, 64, 32, 16, False)
        names = [n for n, _ in h.profile_read()]
    finally:
        h.profile_enable(False)
    assert any("k_prep" in n for n in names), names
    assert any(("k_fused" in n or "k_wgmma" in n) for n in names) == wgmma, names


@pytest.mark.parametrize("neg_head", [False, True])
def test_prep_negative_blocks_rescal(neg_head):
    """RESCAL forms its a-side rows in its own kernel; k_prep runs only the negatives' blocks (partial: Ns = 40)."""
    _check("RESCAL", 64, 12.0, 2000, 20, 192, 64, 40, neg_head, adversarial=False)
