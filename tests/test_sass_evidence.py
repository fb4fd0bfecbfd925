"""The built extension really contains the Hopper instructions the design claims (checked from the cubin with
cuobjdump — no GPU needed): wgmma -> HGMMA, TMA -> UTMALDG (2-D, 4-D, multicast), mbarrier -> SYNCS, multimem.ld_reduce ->
LDGMC, .sys-scope release/acquire flags."""
import glob
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def sass():
    so = sorted(glob.glob(os.path.join(ROOT, "colearn_federated_learning_b200", "ops", "_colearn_C*.so")))
    if not so or shutil.which("cuobjdump") is None:
        pytest.skip("needs the built extension and cuobjdump")
    out = subprocess.run(["cuobjdump", "-sass", so[0]], capture_output=True, text=True, timeout=300)
    if out.returncode != 0 or "Function :" not in out.stdout:
        pytest.skip("cuobjdump could not read the extension")
    per_kernel, cur = {}, None
    for line in out.stdout.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            per_kernel[cur] = []
        elif cur is not None:
            per_kernel[cur].append(line)
    assert "sm_90a" in out.stdout or "SM90" in out.stdout.upper() or per_kernel
    return {k: "\n".join(v) for k, v in per_kernel.items()}


def _kernels(sass, needle):
    return {k: v for k, v in sass.items() if needle in k}


def test_gemm_kernels_use_wgmma_and_tma(sass):
    gemms = _kernels(sass, "gemm_wgmma_kernel")
    assert len(gemms) >= 6                                     # K-major x3 tiles (+cluster), MN-major, mixed, 128x64
    for name, text in gemms.items():
        for mnemonic in ("HGMMA", "UTMALDG", "SYNCS"):
            assert mnemonic in text, (name, mnemonic)
    # implicit-GEMM convolution: 4-D activation boxes in the 1-CTA instantiations
    assert sum("UTMALDG.4D" in t for t in gemms.values()) >= 5
    # the cluster pair multicasts its shared B tile
    assert any("MULTICAST" in t.upper() for t in gemms.values())


def test_comm_kernels_use_multimem_and_system_scope_flags(sass):
    twoshot = next(iter(_kernels(sass, "twoshot_fedavg_kernel").values()))
    assert "LDGMC" in twoshot and "STRONG.SYS" in twoshot      # multimem.ld_reduce + .sys-scope stores / flags
    star = next(iter(_kernels(sass, "star_round_kernel").values()))
    assert "STRONG.SYS" in star
    mlp = _kernels(sass, "mlp_local_sgd_kernel_v2")
    assert mlp and all("STRONG.SYS" in t for t in mlp.values())  # wait / signal flags of the persistent kernel


def test_round2_paths_compile_to_the_instructions_their_docs_claim(sass):
    # programmatic dependent launch: every conv / BatchNorm / pooling kernel exists twice, the PDL twin starts with
    # griddepcontrol.wait / launch_dependents; the plain twin has neither
    conv = {k: v for k, v in sass.items() if re.search(r"(im2col|col2im|bn_apply|bn_bwd|bn_reduce|bn_finalize|maxpool|avgpool|pack|splitk_reduce)\w*kernel", k)}
    with_pdl = [k for k, v in conv.items() if "ACQBULK" in v and "PREEXIT" in v]
    without = [k for k, v in conv.items() if "ACQBULK" not in v and "PREEXIT" not in v]
    assert len(with_pdl) == len(without) == 13, (len(with_pdl), len(without))
    for text in _kernels(sass, "gemm_wgmma_kernel").values():
        assert "ACQBULK" in text and "PREEXIT" in text          # behind `if (ep.pdl)`, after the kernel's own set-up
    # fused wgrad -> FedAvg reduce: the overlapped two-shot polls .sys-scope flags and shares the reduce body
    overlap = next(iter(_kernels(sass, "twoshot_overlap_kernel").values()))
    assert "STRONG.SYS" in overlap and "LDGMC" in overlap
    assert _kernels(sass, "produced_mark_kernel")
    # persistent MLP, variant 5: 128-bit shared-memory loads of the blocked slices; the default variant has none
    v5 = {k: v for k, v in _kernels(sass, "mlp_local_sgd_kernel_v2").items() if "7v2_128b" in k and "Li64ELi64" in k}
    v3 = {k: v for k, v in _kernels(sass, "mlp_local_sgd_kernel_v2").items() if "6v2_128" in k and "Li64ELi64" in k}
    assert len(v5) == 2 and all(t.count("LDS.128") >= 16 for t in v5.values())
    assert len(v3) == 2 and all("LDS.128" not in t for t in v3.values())
    # variant 6: the paired form of variant 5 is built too (Hopper has no packed fp32 FMA, so it issues plain FFMA)
    v6 = {k: v for k, v in _kernels(sass, "mlp_local_sgd_kernel_v2").items() if "7v2_128p" in k and "Li64ELi64" in k}
    assert len(v6) == 2 and all("FFMA" in t for t in v6.values())
    # bounded flag waits: the spin helper reads the nanosecond timer; the comm kernels carry the trap of spin_wait_failed
    star = next(iter(_kernels(sass, "star_round_kernel").values()))
    assert "GLOBALTIMER" in star.upper() or "SR_GLOBALTIMER" in star.upper()
    assert _kernels(sass, "twoshot_resync_kernel") and _kernels(sass, "scale_inplace_kernel")
