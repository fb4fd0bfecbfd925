"""Compile evidence of the layer-wise trainer's local optimizer (no GPU needed), read from the objects and the ptxas -v output
the build keeps: the 8 instances of gemm_wgmma_opt_kernel (tile width 128 / 256 x K-major / MN-major operands x SGD / Adam)
exist, carry the wgmma / TMA / mbarrier pipeline and the programmatic-dependent-launch prologue of gemm_wgmma_kernel, and use
about the local memory of the plain fused-SGD wgrad instance of the same tile and operand form; local_opt_apply_kernel does not
spill and uses no local memory.

The consumer warpgroups of every gemm_wgmma.cu instance live under ptxas's 168-register cap of a 384-thread block (setmaxnreg
raises it only at run time), and the plain 256-wide instances already spill about 1.7 KB per thread there.  The optimizer
instances stay at or below their plain twin's spill, plus at most 48 bytes for the moments of the epilogue (measured: the
128-wide MN-major SGD instance, 80 bytes against 44); the 128-wide K-major SGD instance spills nothing."""
import glob
import os
import re
import shutil
import subprocess

import pytest

from test_local_opt_sass import _local_memory
from test_robust_agg_sass import OBJ, _ptxas

FORMS = [(bn, mn, kind) for bn in (128, 256) for mn in (0, 1) for kind in (1, 2)]


def _opt_name(names, bn, mn, kind):
    hits = [k for k in names if f"gemm_wgmma_opt_kernelILi{bn}ELb{mn}ELi{kind}EE" in k]
    assert len(hits) == 1, (bn, mn, kind, sorted(names))
    return hits[0]


def _plain_name(names, bn, mn):
    hits = [k for k in names if f"17gemm_wgmma_kernelILi{bn}ELi1ELb{mn}ELb{mn}EE" in k]
    assert len(hits) == 1, (bn, mn, sorted(names))
    return hits[0]


def test_optimizer_instances_exist_and_spill_no_more_than_their_plain_twin():
    info = _ptxas("gemm_wgmma.cu")
    assert sum("gemm_wgmma_opt_kernel" in k for k in info) == 8, sorted(info)
    for bn, mn, kind in FORMS:
        spill, _ = info[_opt_name(info, bn, mn, kind)]
        plain, _ = info[_plain_name(info, bn, mn)]
        assert spill <= plain + 48, (bn, mn, kind, spill, plain)
    assert info[_opt_name(info, 128, 0, 1)][0] == 0
    apply = [v for k, v in _ptxas("elementwise.cu").items() if "local_opt_apply_kernel" in k]
    assert len(apply) == 1 and apply[0][0] == 0, apply


def test_optimizer_instances_local_memory():
    lm = _local_memory("gemm_wgmma.cu")
    for bn, mn, kind in FORMS:
        got, plain = lm[_opt_name(lm, bn, mn, kind)], lm[_plain_name(lm, bn, mn)]
        assert got["LDL"] <= plain["LDL"] + 8 and got["STL"] <= plain["STL"] + 4, (bn, mn, kind, got, plain)
    assert lm[_opt_name(lm, 128, 0, 1)] == {"LDL": 0, "STL": 0}
    apply = [v for k, v in _local_memory("elementwise.cu").items() if "local_opt_apply_kernel" in k]
    assert apply == [{"LDL": 0, "STL": 0}], apply


def test_optimizer_instances_keep_the_pipeline_and_the_pdl_prologue():
    objs = glob.glob(os.path.join(OBJ, "gemm_wgmma.cu.*.o"))
    tool = shutil.which("cuobjdump") or os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")
    if not objs or not os.path.exists(tool):
        pytest.skip("needs the build's objects and cuobjdump")
    sass = subprocess.run([tool, "-sass", max(objs, key=os.path.getmtime)], capture_output=True, text=True, check=True).stdout
    per, cur = {}, None
    for line in sass.splitlines():
        m = re.match(r"\s+Function : (\S+)", line)
        if m:
            cur = m.group(1)
            per[cur] = []
        elif cur is not None:
            per[cur].append(line)
    opt = {k: "\n".join(v) for k, v in per.items() if "gemm_wgmma_opt_kernel" in k}
    assert len(opt) == 8, sorted(per)
    for name, text in opt.items():
        for mnemonic in ("HGMMA", "UTMALDG", "SYNCS", "ACQBULK", "PREEXIT"):
            assert mnemonic in text, (name, mnemonic)
