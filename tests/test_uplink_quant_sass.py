"""Compile evidence of the uplink codec (no GPU needed): ptxas reports no spill for any instance of quantize_delta_kernel
(int8 / int4), fedavg_q_kernel (int8 / int4, with and without a server optimizer) and fedavg_q_robust_kernel (register paths
KMAX 4 / 8 / 16 / 32 and the general path, int8 / int4).  Read from the ptxas -v output the build keeps next to its objects."""
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
        out[m.group(1)] = int(spill.group(1)) + int(spill.group(2)) if spill else None
    return out


def test_uplink_kernels_do_not_spill():
    info = _ptxas("elementwise.cu")
    found = {k: v for k, v in info.items() if re.search(r"(quantize_delta_kernel|fedavg_q_kernel|fedavg_q_robust_kernel)I", k)}
    enc = sorted(re.search(r"quantize_delta_kernelILi(\d)EE", k).group(1) for k in found if "quantize_delta_kernel" in k)
    dec = sorted(re.search(r"fedavg_q_kernelILi(\d)ELb([01])EE", k).groups() for k in found if "fedavg_q_kernel" in k)
    rob = sorted(tuple(map(int, re.search(r"fedavg_q_robust_kernelILi(\d+)ELi(\d)EE", k).groups())) for k in found if "q_robust" in k)
    assert enc == ["4", "8"], enc
    assert dec == [("4", "0"), ("4", "1"), ("8", "0"), ("8", "1")], dec
    assert rob == sorted((kmax, bits) for kmax in (0, 4, 8, 16, 32) for bits in (4, 8)), rob
    for name, spill in found.items():
        assert spill == 0, (name, spill)
