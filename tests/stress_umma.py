"""Stress / determinism probe of the wgmma score GEMM (run manually on an H100):
repeats kge_score_neg on fresh random rows and compares with an fp64 evaluation of the same formula."""
import os
import sys

import numpy as np
import torch as th

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "dgl-ke_b200"), os.path.join(ROOT, "oracle")):
    sys.path.insert(0, p)
from dglke_b200 import engine as E, _lib  # noqa: E402

dev = th.device("cuda", 0)
iters = int(sys.argv[1]) if len(sys.argv) > 1 else 12
C, Cs, Ns, D = 5, 200, 200, 400
hp = E.Hyper(model="TransE_l2", hidden_dim=D, gamma=19.9)
_lib.get_handle(0).set_engine(int(os.environ.get("ENGINE", "1")))
g = th.Generator(device=dev).manual_seed(0)
bad_total = 0
for it in range(iters):
    h = (th.rand(C * Cs, D, device=dev, generator=g) - 0.5) * 0.11
    r = (th.rand(C * Cs, D, device=dev, generator=g) - 0.5) * 0.11
    n = (th.rand(C * Ns, D, device=dev, generator=g) - 0.5) * 0.11
    got = E.score_neg(hp, h, r, n, C, Cs, Ns, False)
    got2 = E.score_neg(hp, h, r, n, C, Cs, Ns, False)
    a = (h + r).double().reshape(C, Cs, D)
    b = n.double().reshape(C, Ns, D)
    want = 19.9 - th.cdist(a, b, p=2)
    err = (got.double() - want).abs()
    bad = int((err > 5e-5).sum())
    bad_total += bad
    rep = float((got - got2).abs().max())
    idx = th.nonzero(err > 5e-5)[:6].tolist()
    print("iter %2d max_err %.3e bad %d repeat_diff %.3e %s" % (it, float(err.max()), bad, rep, idx), flush=True)
print("TOTAL_BAD", bad_total)
