"""Compile evidence of the asynchronous apply (no GPU needed): the cubin of elementwise.cu holds fedavg_based_kernel with and
without a server optimizer, fedavg_based_robust_kernel on every register path and the general one, and the distance passes
on BasedRows (dagg_based_*_kernel); ptxas reports no spill for any of them.  Read from the ptxas -v output the build keeps next to its
objects."""
import re

from test_robust_agg_sass import _ptxas


def test_async_apply_kernels_are_built_and_do_not_spill():
    info = _ptxas("elementwise.cu")
    based = {k: v for k, v in info.items() if "BasedRows" in k or "fedavg_based" in k}
    mean = sorted(re.search(r"fedavg_based_kernelILb([01])EE", k).group(1) for k in based if "fedavg_based_kernel" in k)
    assert mean == ["0", "1"], sorted(based)
    kmax = sorted(int(re.search(r"ILi(\d+)EE", k).group(1)) for k in based if "fedavg_based_robust_kernel" in k)
    assert kmax == [0, 4, 8, 16, 32], kmax
    assert sum("dagg_based_apply_kernel" in k for k in based) == 4 and sum("dagg_based_center_kernel" in k for k in based) == 4
    assert sum("dagg_based_dist_kernel" in k for k in based) == 1
    for name, (spill, regs) in based.items():
        assert spill == 0, (name, spill, regs)
