"""CPU tests of the host-side mirror: flag surface vs the reference's own parser, batch/chunk
bookkeeping, graph objects and samplers (no CUDA calls)."""
import os
import sys

import numpy as np
import pytest
import torch as th

from dglke_b200 import utils, graph

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_flag_surface_matches_reference_parser():
    """Every option string, default and type of dglke_train's parser (utils.py:199-297, train.py:40-60), against the
    table read off the reference's own parser and stored under tests/golden (golden_util.reference_result)."""
    import json

    def table(p):
        return {" ".join(a.option_strings): [a.default, a.type.__name__ if a.type else None, a.nargs,
                                             list(a.choices) if a.choices else None, type(a).__name__]
                for a in p._actions if a.option_strings and a.dest != "help"}
    train_flags = ("--gpu", "--mix_cpu_gpu", "--valid", "--rel_part", "--async_update", "--has_edge_importance")

    def from_reference():
        sys.path.insert(0, os.path.join(ROOT, "oracle"))
        import ref_harness as rh
        rh.import_reference()
        import importlib
        ref_utils = importlib.import_module("dglke.utils")
        # train-only flags (train.py:44-60): read from the source since importing dglke.train needs more of DGL
        src = open(os.path.join(rh.REFERENCE_PY, "dglke", "train.py")).read()
        return {"common": table(ref_utils.CommonArgParser()), "train_only": [f for f in train_flags if f in src]}
    from golden_util import reference_result
    want = reference_result("parser_flags", from_reference)
    assert json.loads(json.dumps(table(utils.CommonArgParser()))) == want["common"]
    assert want["train_only"] == list(train_flags)
    for flag in train_flags:
        assert any(flag in a.option_strings for a in utils.ArgParser()._actions)


def test_defaults_worth_knowing():
    a = utils.ArgParser().parse_args([])
    assert (a.hidden_dim, a.batch_size, a.neg_sample_size, a.lr, a.gamma) == (400, 1024, 256, 0.01, 12.0)
    assert (a.regularization_coef, a.regularization_norm, a.loss_genre, a.gpu) == (2e-6, 3, "Logsigmoid", [-1])


def test_multi_gpu_hyper_carries_every_parsed_field():
    """The multi-GPU worker builds its step configuration with train.hyper_from_args: every field of engine.Hyper comes
    from its flag, set here to a value other than the default, so a dropped flag shows up as the default."""
    import dataclasses
    from dglke_b200.engine import Hyper
    from dglke_b200.train import hyper_from_args
    argv = {"model": (["--model_name", "RotatE"], "RotatE"), "hidden_dim": (["--hidden_dim", "72"], 72),
            "gamma": (["--gamma", "7.5"], 7.5), "lr": (["--lr", "0.3"], 0.3),
            "reg_coef": (["--regularization_coef", "3e-5"], 3e-5), "reg_norm": (["--regularization_norm", "2"], 2),
            "adversarial": (["-adv"], True), "adv_temperature": (["-a", "0.4"], 0.4),
            "double_ent": (["-de"], True), "double_rel": (["-dr"], True), "loss_genre": (["--loss_genre", "Hinge"], "Hinge"),
            "margin": (["-m", "2.5"], 2.5), "pairwise": (["-pw"], True), "neg_deg_sample": (["--neg_deg_sample"], True)}
    fields = {f.name: f.default for f in dataclasses.fields(Hyper)}
    assert sorted(argv) == sorted(fields), "a Hyper field without a flag here: extend this test and hyper_from_args"
    hp = hyper_from_args(utils.ArgParser().parse_args(sum((a for a, _ in argv.values()), [])))
    for name, (_, want) in argv.items():
        assert want != fields[name], name
        assert getattr(hp, name) == want, name


def test_multi_gpu_refuses_neg_deg_sample():
    from dglke_b200.train import train_multi_gpu
    args = utils.ArgParser().parse_args(["--gpu", "0", "1", "--neg_deg_sample"])
    with pytest.raises(SystemExit, match="neg_deg_sample"):
        train_multi_gpu(args, 100, 4, (np.zeros(8), np.zeros(8), np.zeros(8)))


def test_batch_size_rounding():
    assert utils.get_compatible_batch_size(1000, 256) == 1024     # utils.py:27-33
    assert utils.get_compatible_batch_size(1024, 256) == 1024
    assert utils.get_compatible_batch_size(100, 256) == 100       # smaller than neg: untouched


def test_chunk_layout_matches_reference_rules():
    assert graph.chunk_layout(1000, 200) == (5, 200)
    assert graph.chunk_layout(100, 256) == (1, 100)               # sampler.py:497-500
    assert graph.chunk_layout(1001, 200) is None                  # ragged: skipped (sampler.py:503-504)


def test_pos_graph_and_sampler():
    pg = graph.build_pos_graph([5, 3, 5], [0, 1, 0], [3, 9, 9])
    assert pg.ndata["id"].tolist() == [3, 5, 9]
    h, t = pg.all_edges(order="eid")
    assert pg.ndata["id"][h].tolist() == [5, 3, 5] and pg.ndata["id"][t].tolist() == [3, 9, 9]
    assert pg.number_of_edges() == 3
    s = graph.SyntheticSampler(100, 7, 12, 4, seed=1)
    p1, n1 = next(s)
    p2, n2 = next(s)
    assert (n1.neg_head, n2.neg_head) == (False, True)           # tail first, then head (sampler.py:853-859)
    assert (n1.num_chunks, n1.chunk_size, n1.neg_sample_size) == (3, 4, 4)
    assert n1.ndata["id"][n1.tail_nid].shape[0] == 12
    p1b, _ = graph.SyntheticSampler(100, 7, 12, 4, seed=1).batch(0)
    assert th.equal(p1.ndata["id"], p1b.ndata["id"])             # seeded => reproducible


def test_triple_sampler_epochs_and_partition():
    rng = np.random.default_rng(0)
    h, r, t = rng.integers(0, 50, 100), rng.integers(0, 3, 100), rng.integers(0, 50, 100)
    s = graph.TripleSampler(h, r, t, 50, 3, 20, 5, seed=2)
    seen = []
    for k in range(5):                                            # one epoch = 5 batches of 20
        pg, ng = s.batch(k)
        hh, tt = pg.all_edges()
        seen += list(zip(pg.ndata["id"][hh].tolist(), pg.edata["id"].tolist(), pg.ndata["id"][tt].tolist()))
    assert sorted(seen) == sorted(zip(h.tolist(), r.tolist(), t.tolist()))
    parts = [graph.TripleSampler(h, r, t, 50, 3, 10, 5, seed=2, rank=k, world=2).n_edges for k in range(2)]
    assert sum(parts) == 100


def test_eval_batches_one_chunk_all_entities():
    b = list(graph.eval_batches(np.array([1, 2, 3]), np.array([0, 0, 1]), np.array([4, 5, 6]), 10, 2, True))
    assert len(b) == 2
    pg, ng = b[0]
    assert (ng.num_chunks, ng.chunk_size, ng.neg_sample_size, ng.neg_head) == (1, 2, 10, True)


def test_lazy_log_and_fused_loss_read_device_scalars_lazily():
    """log dict semantics of the reference (pos_loss, neg_loss, loss, regularization floats; loss excludes reg,
    general_models.py:569-576) on top of the device log4 buffer."""
    from dglke_b200.loss import LazyLog, FusedLoss
    log4 = th.tensor([0.25, 0.75, 0.5, 0.125])
    log = LazyLog(log4, has_reg=True)
    log4.zero_()                                   # the log owns a snapshot
    assert sorted(log.keys()) == ["loss", "neg_loss", "pos_loss", "regularization"]
    assert log["loss"] == 0.5 and log["regularization"] == 0.125 and "pos_loss" in log
    assert sum(l[k] for l in [log, log] for k in ["loss"]) == 1.0      # train loop's averaging idiom
    assert sorted(k for k in LazyLog(th.zeros(4), has_reg=False)) == ["loss", "neg_loss", "pos_loss"]
    loss = FusedLoss(th.tensor([0.25, 0.75, 0.5, 0.125]), with_reg=True)
    assert loss.backward() is None and abs(float(loss) - 0.625) < 1e-7 and loss.item() == float(loss)


def test_loss_generator_argument_errors_match_the_reference():
    """loss.py:58-62, base_loss.py:83-84: the same ValueErrors for the same argument combinations."""
    from dglke_b200.loss import LossGenerator, LazyLog
    for genre in ("Hinge", "Logistic", "Logsigmoid", "BCE"):
        g = LossGenerator(None, genre)
        assert g.neg_label == (0 if genre == "BCE" else -1) and g.pairwise is False
    assert LossGenerator(None, "Hinge", pairwise=True).pairwise and LossGenerator(None, "Logistic", pairwise=True).pairwise
    with pytest.raises(ValueError):
        LossGenerator(None, "Logsigmoid", pairwise=True)
    with pytest.raises(ValueError):
        LossGenerator(None, "BCE", pairwise=True)
    with pytest.raises(ValueError):
        LossGenerator(None, "Hinge", neg_adversarial_sampling=True, pairwise=True)
    with pytest.raises(ValueError):
        LossGenerator(None, "Huber")
    # the pairwise form logs 'loss' (+ 'regularization') only (loss.py:78-80)
    assert sorted(LazyLog(th.zeros(4), has_reg=True, only_loss=True).keys()) == ["loss", "regularization"]
    assert sorted(LazyLog(th.zeros(4), has_reg=False, only_loss=True).keys()) == ["loss"]


def test_unsupported_options_raise_instead_of_falling_back():
    from dglke_b200 import _lib
    with pytest.raises(_lib.KgeError):
        _lib.make_cfg("TransR", 8, 8, 12.0, 0.1, 0.1, 0.0, 3, False, 1.0, False, 8, 8, 8)
    with pytest.raises(ValueError):
        _lib.make_cfg("DistMult", 8, 8, 12.0, 0.1, 0.1, 0.0, 3, False, 1.0, False, 8, 8, 8, loss_genre="Huber")


def test_triple_filter_marks_exactly_the_true_corruptions():
    """Filtered evaluation (sampler.py:514-597 filter_false_neg -> neg_g.edata['bias'] = -1): brute force."""
    from dglke_b200.graph import TripleFilter, eval_batches
    rng = np.random.default_rng(0)
    n_ent, n_rel, n = 50, 4, 600
    h, r, t = rng.integers(0, n_ent, n), rng.integers(0, n_rel, n), rng.integers(0, n_ent, n)
    f = TripleFilter(h, r, t, n_rel)
    known = set(zip(h.tolist(), r.tolist(), t.tolist()))
    for neg_head in (False, True):
        got = f.bias(h[:40], r[:40], t[:40], n_ent, neg_head)
        want = np.zeros((40, n_ent), np.float32)
        for i in range(40):
            for e in range(n_ent):
                if ((e, r[i], t[i]) if neg_head else (h[i], r[i], e)) in known:
                    want[i, e] = -1
        assert np.array_equal(got, want)
        assert all(got[i, (h if neg_head else t)[i]] == -1 for i in range(40))      # the positive's own copy is filtered
        cand = np.sort(rng.choice(n_ent, 20, replace=False))
        assert np.array_equal(f.bias(h[:40], r[:40], t[:40], 20, neg_head, cand), want[:, cand])
    # a triple nobody has seen filters nothing
    assert f.bias([0], [0], [0], n_ent, False).sum() == -sum(1 for e in range(n_ent) if (0, 0, e) in known)
    for pg, ng in eval_batches(h[:10], r[:10], t[:10], n_ent, 4, True, known=f):
        b = ng.edata["bias"]
        assert tuple(b.shape) == (pg.number_of_edges(), n_ent) and b.dtype == th.float32
        assert ng.num_chunks == 1 and ng.neg_sample_size == n_ent
