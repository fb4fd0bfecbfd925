"""Compile evidence of the local optimizer instances (no GPU needed), read from the objects and the ptxas -v output the build
keeps: the 10 instances of mlp_persistent_opt.cu (SGD and Adam for each of the five persistent nets) exist and do not spill,
and their SASS has no local-memory load at all and the same local-memory stores as variant 1's plain kernel of the same net
(the argument buffer of the spin-wait failure report, which every persistent kernel has)."""
import glob
import os
import re
import shutil
import subprocess

import pytest

from test_robust_agg_sass import OBJ, _ptxas

NETS = ["ILb1EJLi10ELi50ELi30ELi10ELi1EEEE", "ILb0EJLi10ELi64ELi64ELi2EEEE", "ILb0EJLi2ELi50ELi10ELi1EEEE",
        "ILb0EJLi10ELi32ELi4ELi32ELi10EEEE", "ILb0EJLi10ELi50ELi30ELi10ELi5EEEE"]


def test_optimizer_instances_exist_and_do_not_spill():
    info = _ptxas("mlp_persistent_opt.cu")
    opt = {k: v for k, v in info.items() if "mlp_local_sgd_opt_kernel" in k}
    assert len(opt) == 10, sorted(info)
    for net in NETS:
        for kind in ("Li1EEEv", "Li2EEEv"):
            assert sum(1 for k in opt if net + kind in k) == 1, (net, kind, sorted(opt))
    for name, (spill, regs) in opt.items():
        assert spill == 0, (name, spill, regs)


def _local_memory(source):
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
            count[cur] = {"LDL": 0, "STL": 0}
        elif cur is not None:
            for op in ("LDL", "STL"):
                if re.search(r"\b" + op + r"\b", line):
                    count[cur][op] += 1
    return count


def test_optimizer_instances_use_no_local_memory():
    opt = {k: v for k, v in _local_memory("mlp_persistent_opt.cu").items() if "mlp_local_sgd_opt_kernel" in k}
    assert len(opt) == 10, sorted(opt)
    plain = {k: v for k, v in _local_memory("mlp_persistent.cu").items() if "20mlp_local_sgd_kernelI" in k}
    for name, c in opt.items():
        assert c["LDL"] == 0, (name, c)
        same_net = [v for k, v in plain.items() if any(net in k and net in name for net in NETS[:3])]
        assert c["STL"] <= max([v["STL"] for v in same_net] + [2]), (name, c)
