"""Compile evidence of the attack-category FFNN's instances (no GPU needed), read from the objects and the ptxas -v output the
build keeps: none of the 8 instances (variants 1, 3, 5, 6 x batch 1 / accumulating where they differ, the forward) spills,
and the fused softmax head leaves the block barriers of the FFNN's kernels as they are.

What is counted is every BAR.SYNC instruction of the whole kernel function, not the barriers one step executes: the step body
is emitted twice in the batch-1 kernels (the first step of a chunk and the steps with deferred updates), and the function also
holds the chunk pipeline's barriers.  Equal counts for the two nets, with the same code around the step loop, mean the same
3 block barriers per step as the FFNN's."""
import glob
import os
import re
import shutil
import subprocess

import pytest

from test_robust_agg_sass import OBJ, _ptxas

CAT = "Li10ELi50ELi30ELi10ELi5E"
FFNN = "Li10ELi50ELi30ELi10ELi1E"


def test_category_instances_do_not_spill():
    info = _ptxas("mlp_persistent_cat.cu")
    cat = {k: v for k, v in info.items() if CAT in k}
    assert len(cat) == 8, sorted(info)                 # v2_128 / 128b / 128p x (plain, accumulate), variant 1, forward
    for name, (spill, regs) in cat.items():
        assert spill == 0, (name, spill, regs)


def _barriers(source):
    objs = glob.glob(os.path.join(OBJ, source + ".*.o"))
    tool = shutil.which("cuobjdump") or os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")
    if not objs or not os.path.exists(tool):
        pytest.skip("needs the build's objects and cuobjdump")
    sass = subprocess.run([tool, "-sass", max(objs, key=os.path.getmtime)], capture_output=True, text=True, check=True).stdout
    count, cur = {}, None
    for line in sass.splitlines():
        m = re.match(r"\s+Function : (\S+)", line)
        if m:
            cur = m.group(1)
            count[cur] = 0
        elif cur is not None and re.search(r"\bBAR\.SYNC", line):
            count[cur] += 1
    return count


@pytest.mark.parametrize("ns", ["v2_128b", "v2_128p"])
@pytest.mark.parametrize("acc", ["Lb0E", "Lb1E"])
def test_softmax_head_keeps_the_ffnn_barriers(ns, acc):
    def pick(counts, net):
        hit = [v for k, v in counts.items() if ns + "23mlp_local_sgd_kernel_v2" in k and net + "EEE" + acc in k]
        assert len(hit) == 1, sorted(counts)
        return hit[0]
    ffnn, cat = pick(_barriers("mlp_persistent.cu"), FFNN), pick(_barriers("mlp_persistent_cat.cu"), CAT)
    assert cat == ffnn, (ns, acc, cat, ffnn)
