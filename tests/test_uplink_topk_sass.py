"""Compile evidence of the top-k uplink (no GPU needed): ptxas reports no spill for topk_delta_kernel and for both instances
of fedavg_topk_kernel (with and without a server optimizer).  Read from the ptxas -v output the build keeps next to its
objects."""
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


def test_topk_kernels_do_not_spill():
    info = _ptxas("elementwise.cu")
    enc = [k for k in info if re.search(r"17topk_delta_kernelE", k)]
    dec = sorted(re.search(r"fedavg_topk_kernelILb([01])EE", k).group(1) for k in info if "fedavg_topk_kernel" in k)
    assert len(enc) == 1, enc
    assert dec == ["0", "1"], dec
    for name in enc + [k for k in info if "fedavg_topk_kernel" in k]:
        assert info[name] == 0, (name, info[name])
