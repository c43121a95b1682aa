"""The compiler's log of kge_rows.cu (written by the build): every instantiation of k_chain and k_update builds without
spilling registers to local memory.

Register counts with CUDA 12.9 for sm_90a (`-Xptxas -v`):
- k_update: 100 registers under __launch_bounds__(256, 2).  Under (256, 4) it was held to 64 registers and spilled its
  loop and staging state inside the row loops.
- k_chain<MODEL, 1>: 48 (TransE_l1), 56 (TransE_l2), 64 (DistMult), 114 (ComplEx), 101 (RotatE).
- k_chain<MODEL, 4> (sharded tables): 104, 104, 121, 114, 101.
RotatE's 32-byte stack frame is the sincosf reduction buffer, not a spill."""
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LOG = os.path.join(ROOT, "dgl-ke_b200", "build", "kge_rows.ptxas.log")

# mangled names: k_update(UpdArgs), k_chain<MODEL, KIT> for the five row models and both load depths
KERNELS = ["_ZN3kge8k_updateENS_7UpdArgsE"] + \
          ["_ZN3kge7k_chainILi%dELi%dEEEvNS_10StepParams" % (m, k) for m in (0, 1, 2, 3, 5) for k in (1, 4)]


@pytest.mark.skipif(not os.path.exists(LOG), reason="no compiler log: the library was not built here")
@pytest.mark.parametrize("kernel", KERNELS)
def test_row_kernel_does_not_spill(kernel):
    log = open(LOG).read()
    blocks = re.split(r"ptxas info\s+: Compiling entry function ", log)
    hit = [b for b in blocks if b.startswith("'") and b.split("'")[1].startswith(kernel)]
    assert len(hit) == 1, "no compiler output for %s" % kernel
    props = hit[0].split("Used")[0]
    assert "0 bytes spill stores, 0 bytes spill loads" in props, (kernel, hit[0][:400])
