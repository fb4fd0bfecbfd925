"""Compile evidence of the robust aggregators (no GPU needed): ptxas reports no spill for any robust instance of the star,
two-shot and overlapped two-shot kernels, nor for fedavg_robust_kernel on its register paths (KMAX 4 / 8 / 16 / 32) and its
general path.  Read from the ptxas -v output the build keeps next to its objects."""
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OBJ = os.path.join(ROOT, "colearn_federated_learning_b200", "ops", "csrc", "_obj")


def _ptxas(source):
    path = os.path.join(OBJ, source + ".log")
    if not os.path.exists(path):
        pytest.skip("needs the build's ptxas log (run the build first)")
    lines = open(path).read().splitlines()
    out = {}
    for i, line in enumerate(lines):
        m = re.search(r"Compiling entry function '(\S+)' for 'sm_90a'", line)
        if not m:
            continue
        block = " ".join(lines[i + 1: i + 4])
        spill = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", block)
        regs = re.search(r"Used (\d+) registers", block)
        out[m.group(1)] = (int(spill.group(1)) + int(spill.group(2)) if spill else None, int(regs.group(1)) if regs else None)
    return out


def test_robust_comm_kernels_do_not_spill():
    info = _ptxas("comm.cu")
    robust = {k: v for k, v in info.items() if re.search(r"(star_round_kernel|twoshot_fedavg_kernel|twoshot_overlap_kernel)ILb[01]ELb1EE", k)}
    assert len(robust) == 6, sorted(info)                      # 3 kernels x (with / without a server optimizer)
    for name, (spill, regs) in robust.items():
        assert spill == 0, (name, spill, regs)


def test_fedavg_robust_kernel_does_not_spill():
    info = _ptxas("elementwise.cu")
    robust = {k: v for k, v in info.items() if "fedavg_robust_kernel" in k}
    kmax = sorted(int(re.search(r"ILi(\d+)EE", k).group(1)) for k in robust)
    assert kmax == [0, 4, 8, 16, 32], kmax
    for name, (spill, regs) in robust.items():
        assert spill == 0, (name, spill, regs)
