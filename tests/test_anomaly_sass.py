"""Compile evidence of federated anomaly detection (no GPU needed): ptxas reports no spill for the autoencoder's instances
of the persistent MLP kernels (variants 1, 3, 5, 6 and the forward) or for recon_summary_kernel.  Read from the ptxas -v
output the build keeps next to its objects."""
from test_robust_agg_sass import _ptxas


def test_autoencoder_instances_do_not_spill():
    info = _ptxas("mlp_persistent_ae.cu")
    ae = {k: v for k, v in info.items() if "Li10ELi32ELi4ELi32ELi10E" in k}
    assert len(ae) == 8, sorted(info)                      # v2_128 / 128b / 128p x (plain, accumulate), variant 1, forward
    assert not any("Li64ELi64" in k for k in info)         # the MLP64 selector of test_sass_evidence.py never sees them
    for name, (spill, regs) in ae.items():
        assert spill == 0, (name, spill, regs)


def test_recon_summary_kernel_does_not_spill():
    info = _ptxas("elementwise.cu")
    inst = {k: v for k, v in info.items() if "recon_summary_kernel" in k}
    assert len(inst) == 1, sorted(info)
    for name, (spill, regs) in inst.items():
        assert spill == 0, (name, spill, regs)
