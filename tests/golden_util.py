"""Helpers shared by the CPU (oracle-vs-golden) and GPU (CUDA-vs-golden) parity tests."""
import glob
import json
import os

import numpy as np
import torch as th

GOLDEN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def golden_cases():
    return sorted(os.path.splitext(os.path.basename(p))[0] for p in glob.glob(os.path.join(GOLDEN_DIR, "*.npz")))


def load_case(name):
    z = np.load(os.path.join(GOLDEN_DIR, name + ".npz"))
    meta = json.loads(str(z["meta"]))
    return meta, z


def hyper_from_meta(meta):
    import kge_oracle as ko
    return ko.Hyper(model=meta["model"], hidden_dim=meta["hidden_dim"], gamma=meta["gamma"], lr=meta["lr"],
                    reg_coef=meta["reg_coef"], reg_norm=meta["reg_norm"], adversarial=meta["adversarial"],
                    adv_temperature=meta["adv_temperature"], double_ent=meta["double_ent"],
                    double_rel=meta["double_rel"], loss_genre=meta.get("loss_genre", "Logsigmoid"),
                    margin=meta.get("margin", 1.0), pairwise=meta.get("pairwise", False),
                    neg_deg_sample=meta.get("neg_deg_sample", False))


def step_inputs(z, step):
    p = "s%d_" % step
    t = lambda k: th.from_numpy(np.ascontiguousarray(z[p + k]))
    d = dict(node_ids=t("node_ids"), head_local=t("head_local"), tail_local=t("tail_local"),
             rel_ids=t("rel_ids"), neg_ids=t("neg_ids"), neg_head=bool(int(z[p + "neg_head"])))
    d["edge_weight"] = t("edge_weight") if (p + "edge_weight") in z.files else None
    return d


def tables_before(z, step):
    """(ent_emb, ent_state, rel_emb, rel_state) the reference held BEFORE `step` (fresh copies)."""
    f = lambda a: th.from_numpy(np.array(a, copy=True))
    if step == 0:
        ent, rel = f(z["ent_emb0"]), f(z["rel_emb0"])
        return ent, th.zeros(ent.shape[0]), rel, th.zeros(rel.shape[0])
    p = "s%d_" % (step - 1)
    return f(z[p + "ent_emb"]), f(z[p + "ent_state"]), f(z[p + "rel_emb"]), f(z[p + "rel_state"])


REF_HOST = os.path.join(GOLDEN_DIR, "reference_host.json.gz")


def reference_result(key, make):
    """What the unmodified reference returned for `key` (dataset readers, parser tables): stored in
    tests/golden/reference_host.json.gz.  With KGE_WRITE_GOLDEN=1 (and a checkout of the reference, see
    oracle/ref_harness.py) make() is run on the reference instead: a new key is stored, an existing one must match."""
    import gzip
    db = json.load(gzip.open(REF_HOST, "rt")) if os.path.exists(REF_HOST) else {}
    if os.environ.get("KGE_WRITE_GOLDEN") == "1":
        data = json.loads(json.dumps(make()))
        assert db.setdefault(key, data) == data, key
        with gzip.GzipFile(REF_HOST, "wb", mtime=0) as f:
            f.write(json.dumps(db, sort_keys=True).encode())
    return db[key]
