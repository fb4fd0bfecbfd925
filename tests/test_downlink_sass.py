"""Compile evidence of the compressed downlink (no GPU needed): ptxas reports no spill for the six new kernel instances
(downlink_quant_kernel and replica_apply_q_kernel for int8 and int4, downlink_topk_kernel, replica_apply_topk_kernel).
Read from the ptxas -v output the build keeps next to its objects."""
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


def test_downlink_kernels_do_not_spill():
    info = _ptxas("elementwise.cu")
    found = {}
    for pat in (r"21downlink_quant_kernelILi8E", r"21downlink_quant_kernelILi4E", r"20downlink_topk_kernelE",
                r"22replica_apply_q_kernelILi8E", r"22replica_apply_q_kernelILi4E", r"25replica_apply_topk_kernelE"):
        names = [k for k in info if re.search(pat, k)]
        assert len(names) == 1, (pat, names)
        found[names[0]] = info[names[0]]
    assert all(v == 0 for v in found.values()), found
