"""The buffers a handle keeps between steps (step workspace, relation sums, --neg_deg_sample id list, staging of the
host entry point): steps captured into a CUDA graph after an eager one, growth refused inside a capture, and regrowth
when the shape changes between eager steps."""
import numpy as np
import pytest
import torch as th

import kge_oracle as ko

pytestmark = pytest.mark.gpu

N_ENT, N_REL = 3000, 20


def _batch(B, Cs, Ns, seed):
    rng = np.random.default_rng(seed)
    h, t = rng.integers(0, N_ENT, B), rng.integers(0, N_ENT, B)
    nodes, inv = np.unique(np.concatenate([h, t]), return_inverse=True)
    T = lambda a: th.from_numpy(np.ascontiguousarray(a.astype(np.int64)))
    return [T(nodes), T(inv[:B]), T(inv[B:]), T(rng.integers(0, N_REL, B)), T(rng.integers(0, N_ENT, B // Cs * Ns))]


def _hyper(neg_deg_sample=False):
    return ko.Hyper(model="TransE_l2", hidden_dim=64, gamma=12.0, lr=0.1, reg_coef=1e-6, adversarial=True,
                    neg_deg_sample=neg_deg_sample)


def _engine(hp, tables, handle=None):
    """A StepEngine on a handle of its own (or on `handle`): the buffers under test start empty."""
    from dglke_b200 import _lib
    from dglke_b200.engine import StepEngine, DeviceTable, Hyper
    hyper = Hyper(model=hp.model, hidden_dim=hp.hidden_dim, gamma=hp.gamma, lr=hp.lr, reg_coef=hp.reg_coef,
                  adversarial=hp.adversarial, neg_deg_sample=hp.neg_deg_sample)
    eng = StepEngine(hyper, DeviceTable.from_tensors(tables[0], tables[1]), DeviceTable.from_tensors(tables[2], tables[3]), 0)
    eng.h = handle if handle is not None else _lib.Handle(0)
    return eng


def _device_tables(tables):
    return [x.to(th.device("cuda", 0)).contiguous() for x in tables]


def _oracle_step(hp, o, si, Cs, Ns, neg_head):
    return ko.train_step(hp, o[0], o[1], o[2], o[3], *si, len(si[1]) // Cs, Cs, Ns, neg_head)


def _check_tables(dev_tables, want, rtol, atol):
    for got, w, what in zip(dev_tables, want, ("entity", "entity state", "relation", "relation state")):
        np.testing.assert_allclose(got.cpu().numpy(), w.numpy(), rtol=rtol, atol=atol, err_msg=what)


def test_graph_captured_steps_match_eager_steps():
    hp = _hyper()
    tables = ko.init_tables(hp, N_ENT, N_REL, seed=4)
    B, Cs, Ns = 256, 64, 64
    batches = [[x.cuda() for x in _batch(B, Cs, Ns, seed=30 + k)] for k in range(3)]
    te, tg = _device_tables(tables), _device_tables(tables)
    eager, graphed = _engine(hp, te), _engine(hp, tg)
    step = lambda eng, k: eng.step(*batches[k], Cs, Ns, k == 2)
    step(eager, 0)
    step(graphed, 0)                  # the eager step sizes every buffer the captured ones use
    th.cuda.synchronize()
    graphs = {}
    for k in (1, 2):
        graphs[k] = th.cuda.CUDAGraph()
        with th.cuda.graph(graphs[k]):
            step(graphed, k)
    for k in (1, 2, 1, 2):
        graphs[k].replay()
        step(eager, k)
    th.cuda.synchronize()
    # the same kernels on the same inputs; only the order of the float atomics (node gradients, relation sums) differs
    for got, want, what in zip(tg, te, ("entity", "entity state", "relation", "relation state")):
        got, want = got.cpu().numpy(), want.cpu().numpy()
        np.testing.assert_allclose(got, want, rtol=1e-5, atol=1e-5 * float(np.abs(want).max()), err_msg=what)


def test_growing_the_neg_deg_id_list_inside_a_capture_is_refused():
    from dglke_b200 import _lib
    hp, hp_nd = _hyper(), _hyper(neg_deg_sample=True)
    tables = ko.init_tables(hp, N_ENT, N_REL, seed=6)
    dt = _device_tables(tables)
    plain = _engine(hp, dt)
    nd = _engine(hp_nd, dt, handle=plain.h)
    o = [x.clone() for x in tables]
    # a larger plain step leaves a workspace that the smaller --neg_deg_sample step fits, but no id list
    big = _batch(1024, 128, 128, seed=40)
    plain.step(*(x.cuda() for x in big), 128, 128, False)
    _oracle_step(hp, o, big, 128, 128, False)
    th.cuda.synchronize()
    small = _batch(128, 32, 32, seed=41)
    small_dev = [x.cuda() for x in small]
    th.cuda.synchronize()
    g = th.cuda.CUDAGraph()
    with pytest.raises(_lib.KgeError, match="run one eager step first"):
        with th.cuda.graph(g):
            nd.step(*small_dev, 32, 32, False)
    del g
    log = nd.step(*small_dev, 32, 32, False).cpu().numpy()
    fb = _oracle_step(hp_nd, o, small, 32, 32, False)
    np.testing.assert_allclose(log[2], fb["log"]["loss"], rtol=5e-5)
    _check_tables(dt, o, rtol=1e-4, atol=5e-5)


def test_buffers_regrow_across_eager_steps_of_changing_shape():
    """small -> large -> small -> large, each through the device-index entry point and through the pageable host one:
    the workspace and the host staging grow twice and the node-gradient region is re-zeroed past its old extent."""
    hp = _hyper()
    tables = ko.init_tables(hp, N_ENT, N_REL, seed=8)
    dt = _device_tables(tables)
    eng = _engine(hp, dt)
    o = [x.clone() for x in tables]
    shapes = [(64, 32, 32), (512, 128, 128)] * 2
    for k, (B, Cs, Ns) in enumerate(shapes):
        for host in (False, True):
            neg_head = host
            si = _batch(B, Cs, Ns, seed=50 + 2 * k + host)
            if host:
                log = eng.step_host(*si, Cs, Ns, neg_head)
                eng.sync()
            else:
                log = eng.step(*(x.cuda() for x in si), Cs, Ns, neg_head)
            fb = _oracle_step(hp, o, si, Cs, Ns, neg_head)
            np.testing.assert_allclose(log.cpu().numpy()[2], fb["log"]["loss"], rtol=5e-5, err_msg="step %d %s" % (k, host))
    _check_tables(dt, o, rtol=2e-4, atol=1e-6)
