"""Step increments under an environment switch that the library reads once per process (KGE_B200_NO_COOP: the
three-launch k_update; KGE_B200_NO_BULKRED: per-lane red.add instead of cp.reduce.async.bulk).  Run as a script by
tests/test_gpu_step_increments.py with the switch set; prints STEP_INCREMENTS_ENV_OK when every case held."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "tests"), os.path.join(ROOT, "dgl-ke_b200"), os.path.join(ROOT, "oracle")):
    sys.path.insert(0, p)


def main():
    import test_gpu_step_increments as T
    from dglke_b200 import _lib
    env = [k for k in ("KGE_B200_NO_COOP", "KGE_B200_NO_BULKRED") if os.environ.get(k)]
    assert env, "no environment switch set"
    h = _lib.get_handle(0)
    h.profile_enable(True)
    for case in T.ENV_CASES:
        for neg_head in (False, True):
            h.profile_read()
            T.run_fused_case(case, neg_head, "%s %s %s" % ("+".join(env), case.name, "head" if neg_head else "tail"))
            names = [n for n, _ in h.profile_read()]
            if "KGE_B200_NO_COOP" in env:      # the update ran as three launches, not the cooperative one
                assert {"k_update<nodes>", "k_update<state adds>", "k_update<apply>"} <= set(names), names
    print("STEP_INCREMENTS_ENV_OK")


if __name__ == "__main__":
    main()
