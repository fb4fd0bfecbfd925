"""Compile evidence of the class-weighted instances (no GPU needed), read from the objects and the ptxas -v output the build
keeps: the 4 instances of mlp_persistent_cw.cu (variant 5, batch 1 and accumulating, for the FFNN and the attack-category net)
exist and do not spill, and the class weights add no block barrier: every weighted kernel has the BAR.SYNC count of its
unweighted counterpart (counted over the whole function, as test_category_sass.py explains)."""
import pytest

from test_category_sass import CAT, FFNN, _barriers
from test_robust_agg_sass import _ptxas


def test_weighted_instances_exist_and_do_not_spill():
    info = _ptxas("mlp_persistent_cw.cu")
    cw = {k: v for k, v in info.items() if "mlp_local_sgd_kernel_v2_cw" in k}
    assert len(cw) == 4, sorted(info)
    for net in (FFNN, CAT):
        for acc in ("Lb0E", "Lb1E"):
            assert sum(1 for k in cw if "v2_128b" in k and net + "EEE" + acc in k) == 1, (net, acc, sorted(cw))
    for name, (spill, regs) in cw.items():
        assert spill == 0, (name, spill, regs)


@pytest.mark.parametrize("net,source", [(FFNN, "mlp_persistent.cu"), (CAT, "mlp_persistent_cat.cu")])
@pytest.mark.parametrize("acc", ["Lb0E", "Lb1E"])
def test_weighted_kernels_keep_the_barriers(net, source, acc):
    def pick(counts, kernel):
        hit = [v for k, v in counts.items() if "v2_128b" + kernel in k and net + "EEE" + acc in k]
        assert len(hit) == 1, sorted(counts)
        return hit[0]
    plain = pick(_barriers(source), "23mlp_local_sgd_kernel_v2I")
    weighted = pick(_barriers("mlp_persistent_cw.cu"), "26mlp_local_sgd_kernel_v2_cwI")
    assert weighted == plain, (net, acc, weighted, plain)
