"""Float64 restatement of the inference scores (score_fun.py of the reference, as ScoreInfer uses them) over the full
H x R x T cube, and the brute-force top-K lists of the prediction tests.  Helpers of test_predict_host.py and
test_gpu_predict.py."""
import numpy as np


def cube64(model, ent, rel, H, R, T, gamma, hidden_dim, triplet_wise=False):
    """(scores, error scales) in float64: [nH, nR, nT], or [n] with triplet_wise.  The scale is what
    test_gpu_eval_scores.allowed_error expects: sum |a_k| |b_k| for the bilinear models, |a|^2 + |b|^2 for TransE_l2,
    the distance for TransE_l1 and RotatE."""
    e, r = np.asarray(ent, np.float64), np.asarray(rel, np.float64)
    h, rr, t = e[np.asarray(H)], r[np.asarray(R)], e[np.asarray(T)]
    if triplet_wise:
        h, rr, t = h[:, None, None, :], rr[:, None, None, :], t[:, None, None, :]
    else:
        h, rr, t = h[:, None, None, :], rr[None, :, None, :], t[None, None, :, :]
    if model in ("TransE", "TransE_l2", "TransE_l1"):
        d = h + rr - t
        if model == "TransE_l1":
            dist = np.abs(d).sum(-1)
            s, sc = gamma - dist, dist
        else:
            dist = np.sqrt((d * d).sum(-1))
            a = h + rr
            s, sc = gamma - dist, (a * a).sum(-1) + (t * t).sum(-1)
    elif model == "DistMult":
        s, sc = (h * rr * t).sum(-1), np.abs(h * rr * t).sum(-1)
    elif model == "ComplEx":
        D = h.shape[-1] // 2
        hr, hi, rr_, ri, tr, ti = h[..., :D], h[..., D:], rr[..., :D], rr[..., D:], t[..., :D], t[..., D:]
        s = (hr * rr_ * tr + hi * rr_ * ti + hr * ri * ti - hi * ri * tr).sum(-1)
        sc = (np.abs(hr * rr_ * tr) + np.abs(hi * rr_ * ti) + np.abs(hr * ri * ti) + np.abs(hi * ri * tr)).sum(-1)
    elif model == "RESCAL":
        D = h.shape[-1]
        M = rr.reshape(rr.shape[:-1] + (D, D))
        mt = (M * t[..., None, :]).sum(-1)                        # M_r t
        s = (h * mt).sum(-1)
        sc = (np.abs(h) * (np.abs(M) * np.abs(t)[..., None, :]).sum(-1)).sum(-1)
    elif model == "RotatE":
        D = h.shape[-1] // 2
        emb_init = (gamma + 2.0) / hidden_dim
        ph = rr / (emb_init / np.pi)
        c, sn = np.cos(ph), np.sin(ph)
        hr, hi, tr, ti = h[..., :D], h[..., D:], t[..., :D], t[..., D:]
        re = hr * c - hi * sn - tr
        im = hr * sn + hi * c - ti
        dist = np.sqrt(re * re + im * im).sum(-1)
        s, sc = gamma - dist, dist
    else:
        raise ValueError(model)
    if triplet_wise:
        s, sc = s[:, 0, 0], sc[:, 0, 0]
    return s, sc


def list_keys(exec_mode, nH, nR, nT):
    """(list index, key) of every element of the cube, flattened in (i, j, k) order (triplet_wise: the n triples)."""
    if exec_mode == "triplet_wise":
        return np.zeros(nH, np.int64), np.arange(nH, dtype=np.int64)
    i, j, k = np.meshgrid(np.arange(nH), np.arange(nR), np.arange(nT), indexing="ij")
    key = ((i * nR + j) * nT + k).ravel()
    g = {"all": np.zeros_like(i), "batch_head": i, "batch_rel": j, "batch_tail": k}[exec_mode].ravel()
    return g.astype(np.int64), key.astype(np.int64)


def brute_topk(scores, groups, keys, G, K):
    """[G, K] (scores, keys) of a host sort by (score descending, key ascending), NaN left out, -inf / -1 padded."""
    scores, groups, keys = np.asarray(scores).ravel(), np.asarray(groups).ravel(), np.asarray(keys).ravel()
    out_s = np.full((G, K), -np.inf, dtype=scores.dtype)
    out_k = np.full((G, K), -1, dtype=np.int64)
    ok = ~np.isnan(scores)
    scores, groups, keys = scores[ok], groups[ok], keys[ok]
    o = np.lexsort((keys, -scores, groups))
    scores, groups, keys = scores[o], groups[o], keys[o]
    starts = np.searchsorted(groups, np.arange(G), "left")
    ends = np.searchsorted(groups, np.arange(G), "right")
    for g in range(G):
        n = min(K, ends[g] - starts[g])
        out_s[g, :n] = scores[starts[g]:starts[g] + n]
        out_k[g, :n] = keys[starts[g]:starts[g] + n]
    return out_s, out_k
