"""Federated anomaly detection on the H100: the autoencoder's persistent-kernel variants 1, 3, 5 and 6 against float64
(variant 6 gives variant 5's bits, two launches give the same bits), recon_summary_kernel against the reference bit for bit
at the edges of tests/test_anomaly.py and at 10^6 random rows (the reference equals the SIMT build bit for bit there), and a
local-mode run on the GPU."""
import numpy as np
import pytest
import torch

from colearn_federated_learning_b200 import ops
from colearn_federated_learning_b200.ops import _ext
from colearn_federated_learning_b200.ops import reference as R
import test_mlp_kernel_edges as E
from test_anomaly import check_local, local_run, make_recon_case, offsets_of, same_result, segments_for, ae_fit_case

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")


@pytest.mark.parametrize("n,B", [(0, 1), (1, 1), (65, 1), (1000, 1), (70, 32), (200, 32)])
def test_autoencoder_fit_matches_float64_gpu(n, B):
    res = ae_fit_case(E.Device(), "gpu ae", n, B, 1 if B == 1 else 2, (5, 1, 3, 6))
    assert torch.equal(res[5][0], res[6][0]) and torch.equal(res[5][1], res[6][1]), "variant 6 != 5"
    again = ae_fit_case(E.Device(), "gpu ae", n, B, 1 if B == 1 else 2, (5,))
    assert torch.equal(again[5][0], res[5][0]) and torch.equal(again[5][1], res[5][1]), "two launches differ"


def test_autoencoder_forward_gpu():
    E._forward(E.Device(), "autoencoder", (1, 263, 265, 5000))


def gpu_summary(xh, x, y, segs, B, j, grid=0):
    lab = None if y is None else y.to(DEV)
    c, s, e, f = _ext.require().recon_summary(xh.to(DEV), x.to(DEV), lab, offsets_of(segs), B, -1 if j is None else j, grid)
    torch.cuda.synchronize()
    return c.cpu(), s.cpu(), (e.cpu() if j is not None else None), (f.cpu() if j is not None else None)


@pytest.mark.parametrize("N", [0, 1, 2047, 2048, 2049, 5000])
@pytest.mark.parametrize("B", [32, 256, 4096])
def test_recon_summary_matches_the_reference_gpu(N, B):
    xh, x, y = make_recon_case(N, 7 * N + B)
    segs = segments_for(N)
    j = B // 2 + 3
    got = gpu_summary(xh, x, y, segs, B, j)
    same_result(got, R.recon_summary(xh, x, y, B, offsets_of(segs).tolist(), j))
    same_result(gpu_summary(xh, x, None, segs, B, None), R.recon_summary(xh, x, None, B, offsets_of(segs).tolist())[:2] + (None, None))
    same_result(gpu_summary(xh, x, y, segs, B, j), got)                                    # two launches: the same bits


def test_recon_summary_a_million_rows_and_grids_gpu():
    N = 1_000_000
    xh, x, y = make_recon_case(N, 11)
    segs = [300_000, 0, 1, 699_999]
    ref = R.recon_summary(xh, x, y, 1024, offsets_of(segs).tolist(), 700)
    base = gpu_summary(xh, x, y, segs, 1024, 700)
    same_result(base, ref)
    for grid in (1, 7, 132, 4096):
        same_result(gpu_summary(xh, x, y, segs, 1024, 700, grid), base)
    c, s, e, f = ops.recon_summary(xh.to(DEV), x.to(DEV), y.to(DEV), 1024, segs, 700)
    assert torch.equal(c.cpu(), base[0]) and torch.equal(f.cpu(), base[3])


def test_local_run_on_the_gpu(tmp_path):
    _, recs, meta = local_run(tmp_path, device=DEV)
    check_local(recs, meta)
