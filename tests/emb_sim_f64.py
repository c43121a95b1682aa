"""Float64 restatement of the reference's similarity functions (models/pytorch/tensor_models.py:59-100, as EmbSimInfer
uses them), their fp32 error bounds, and the list keys of the embedding-similarity tests.  Helpers of
test_emb_sim_host.py and test_gpu_emb_sim.py."""
import math

import numpy as np

U = 2.0 ** -24                  # unit roundoff of fp32
C_SUM = 4.0                     # the sqrt(D) constant of test_gpu_eval_scores.allowed_error


def sim64(func, X, Y, pairwise=False):
    """(scores, bounds) in float64: [nL, nR], or [n] with pairwise.  The bound is the largest |fp32 score - float64
    score| an fp32 evaluation may show, per element:

      dot          C_SUM sqrt(D) u sum|x_k y_k| + (3 ceil(D/8) 2^-23 + 4u) |s|, the bilinear bound of
                   test_gpu_eval_scores.allowed_error (the second term covers the 3xTF32 tensor-core accumulation, which
                   rounds toward zero);
      cosine       the dot bound over |x| |y|, plus (C_SUM sqrt(D) + 6) u |s| for the two norms (sums of squares, one
                   sign: C_SUM sqrt(D) u relative, halved by the square root) and the division;
      ext_jaccard  (e_dot + |s| e_den) / den + 2u |s|, with e_den = e_dot + (C_SUM sqrt(D) + 6) u (|x|^2 + |y|^2);
                   den >= (|x|^2 + |y|^2) / 2, so the quotient is well conditioned;
      l1, l2       (C_SUM sqrt(D) + 4) u d: in difference form every term |x_k - y_k| (or its square) is exact to a few
                   u of itself and all have one sign, so the error is proportional to the distance d itself (the
                   expanded form |x|^2 + |y|^2 - 2 x.y has one proportional to |x|^2 + |y|^2 instead)."""
    x, y = np.asarray(X, np.float64), np.asarray(Y, np.float64)
    if not pairwise:
        x, y = x[:, None, :], y[None, :, :]
    D = x.shape[-1]
    k = C_SUM * U * math.sqrt(D)
    if func in ("l1", "l2"):
        d = x - y
        dist = np.abs(d).sum(-1) if func == "l1" else np.sqrt((d * d).sum(-1))
        return -dist, (k + 4 * U) * dist
    dot = (x * y).sum(-1)
    e_dot = k * np.abs(x * y).sum(-1) + (3 * ((D + 7) // 8) * 2 * U + 4 * U) * np.abs(dot)
    if func == "dot":
        return dot, e_dot
    nx, ny = np.sqrt((x * x).sum(-1)), np.sqrt((y * y).sum(-1))
    if func == "cosine":
        s = dot / (nx * ny)
        return s, e_dot / (nx * ny) + (k + 6 * U) * np.abs(s)
    if func == "ext_jaccard":
        sq = nx * nx + ny * ny
        den = sq - dot
        s = dot / den
        e_den = e_dot + (k + 6 * U) * sq
        return s, (e_dot + np.abs(s) * e_den) / den + 2 * U * np.abs(s)
    raise ValueError(func)


def list_keys(exec_mode, nL, nR):
    """(list index, key) of every element, flattened in (i, j) order (pairwise: the n pairs)."""
    if exec_mode == "pairwise":
        return np.zeros(nL, np.int64), np.arange(nL, dtype=np.int64)
    i, j = np.meshgrid(np.arange(nL), np.arange(nR), indexing="ij")
    g = i if exec_mode == "batch_left" else np.zeros_like(i)
    return g.ravel().astype(np.int64), (i * nR + j).ravel().astype(np.int64)
