"""Compile evidence of secure aggregation (no GPU needed): ptxas reports no spill for secagg_mask_kernel,
secagg_streams_kernel and both instances of fedavg_secagg_kernel (with and without a server optimizer).  Read from the ptxas
-v output the build keeps next to its objects."""
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


def test_secagg_kernels_do_not_spill():
    info = _ptxas("elementwise.cu")
    mask = [k for k in info if re.search(r"18secagg_mask_kernelE", k)]
    streams = [k for k in info if re.search(r"21secagg_streams_kernelE", k)]
    apply = sorted(re.search(r"fedavg_secagg_kernelILb([01])EE", k).group(1) for k in info if "fedavg_secagg_kernel" in k)
    assert len(mask) == 1 and len(streams) == 1, (mask, streams)
    assert apply == ["0", "1"], apply
    for name in mask + streams + [k for k in info if "fedavg_secagg_kernel" in k]:
        assert info[name] == 0, (name, info[name])
