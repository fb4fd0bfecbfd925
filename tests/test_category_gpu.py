"""Attack categorisation on the H100: the attack-category FFNN's persistent-kernel instances (variants 5, 6, 3, 1) against
float64 over the same matrix as the SIMT tests in test_category.py, larger; variant 6 = variant 5 and two launches give the
same bits; the batched forward; one local-mode training to the macro-F1 threshold.  Each case records its largest error as
a fraction of its bound (printed at module end with -s)."""
import pytest
import torch

import test_mlp_kernel_edges as E
from test_category import CAT, cat_net, check_local, fit_case, local_run, many_clients, saturated  # noqa: F401 (cat_net: fixture)

gpu = pytest.mark.gpu
device = E.device
_report = E._report_fractions


@gpu
@pytest.mark.parametrize("n", E.BATCH1_N)
def test_batch1_chunk_edges_gpu(device, n):
    fit_case(device, "cat gpu b1", n, 1, 1, -1, (5, 6, 3, 1), bits_pairs=True)


@gpu
@pytest.mark.parametrize("B", E.BATCHES)
def test_batches_gpu(device, B):
    for n in (203, B, B + 5, 0):
        fit_case(device, "cat gpu batch", n, B, 2, -1, (5, 6, 3, 1), bits_pairs=True)


@gpu
@pytest.mark.parametrize("B,n,epochs,max_b", [(1, 100, 3, 150), (7, 100, 3, 20), (1, 100, 2, 100)])
def test_max_batches_gpu(device, B, n, epochs, max_b):
    fit_case(device, "cat gpu max_b", n, B, epochs, max_b, (5, 6, 3, 1), bits_pairs=True)


@gpu
@pytest.mark.parametrize("B", [1, 7])
def test_clients_in_one_launch_gpu(device, B):
    many_clients(device, B, 40, (5, 1))


@gpu
@pytest.mark.parametrize("scale", [20, 60, 100])
def test_saturated_logits_gpu(device, scale):
    saturated(device, scale, (5, 6, 3, 1))


@gpu
@pytest.mark.parametrize("what", ["x_nan", "x_inf", "x_-inf"])
def test_non_finite_features_gpu(device, what):
    E._non_finite(device, CAT, "xent", what, (5, 6, 3, 1))


@gpu
def test_forward_gpu(device):
    E._forward(device, CAT, (1, 263, 264, 265, 100_003))


@gpu
def test_local_training_gpu(tmp_path):
    _, recs, meta = local_run(tmp_path, device=torch.device("cuda", 0))
    check_local(recs, meta)
