"""Compile evidence of the detection-metrics summary (no GPU needed): ptxas reports no spill for either eval_summary_kernel
instance (C = 1 and C >= 2).  Read from the ptxas -v output the build keeps next to its objects."""
import re

from test_robust_agg_sass import _ptxas


def test_eval_summary_kernel_does_not_spill():
    info = _ptxas("elementwise.cu")
    inst = {k: v for k, v in info.items() if "eval_summary_kernel" in k}
    assert sorted(re.search(r"ILb([01])EE", k).group(1) for k in inst) == ["0", "1"], sorted(info)
    for name, (spill, regs) in inst.items():
        assert spill == 0, (name, spill, regs)
