"""The compiler's log of kge_topk.cu (written by the build): both top-K kernels build without spilling registers to
local memory.  With CUDA 12.9 for sm_90a (`-Xptxas -v`) each uses 40 registers; k_topk_select holds 33 KB of static
shared memory (the 4 096 images of a segment and the radix histogram), k_topk_merge 24 KB (the 2 048-entry buffer)."""
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LOG = os.path.join(ROOT, "dgl-ke_b200", "build", "kge_topk.ptxas.log")

KERNELS = ["_ZN3kge13k_topk_selectENS_10TopkParamsE", "_ZN3kge12k_topk_mergeENS_10TopkParamsE"]


@pytest.mark.skipif(not os.path.exists(LOG), reason="no compiler log: the library was not built here")
@pytest.mark.parametrize("kernel", KERNELS)
def test_topk_kernel_does_not_spill(kernel):
    log = open(LOG).read()
    blocks = re.split(r"ptxas info\s+: Compiling entry function ", log)
    hit = [b for b in blocks if b.startswith("'") and b.split("'")[1] == kernel]
    assert len(hit) == 1, "no compiler output for %s" % kernel
    assert "0 bytes spill stores, 0 bytes spill loads" in hit[0].split("Used")[0], hit[0][:400]
