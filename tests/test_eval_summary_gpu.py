"""The detection-metrics summary on the H100: ``ops.eval_summary`` (eval_summary_kernel) against the reference over the same
matrix as the SIMT build in tests/test_fed_eval.py — counts exact, loss to rtol 1e-6 — plus: two calls give identical bits,
launch grids do not change a bit, a 100-segment launch equals 100 single-segment launches, and a model's federated summary
through the GPU forward equals the reference summary of the same outputs."""
import numpy as np
import pytest
import torch

from colearn_federated_learning_b200 import ops
from colearn_federated_learning_b200.fl import fedeval
from colearn_federated_learning_b200.ops import _ext, reference
from test_fed_eval import make_case, segments_for

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")


def _same(a, b):
    return torch.equal(a.view(torch.int64), b.view(torch.int64))


def _check(s, y, B, segs, thr=0.5):
    c1, l1 = ops.eval_summary(s.to(DEV), y.to(DEV), B, thr, segs)
    offs = [0] + np.cumsum(segs).tolist()
    c2, l2 = reference.eval_summary(s, y, B, thr, offs)
    assert torch.equal(c1.cpu(), c2)
    assert torch.allclose(l1.cpu(), l2, rtol=1e-6, atol=0)
    return c1, l1


@pytest.mark.parametrize("C", [1, 2, 10])
@pytest.mark.parametrize("N", [0, 1, 2047, 2048, 2049, 20000])
@pytest.mark.parametrize("B", [2, 256, 4096])
def test_kernel_matches_the_reference(C, N, B):
    if C * 2 * B > 32768:
        pytest.skip("outside the summary's limits (a refusal)")
    s, y = make_case(C, N, 10 * C + N % 7)
    c1, l1 = _check(s, y, B, segments_for(N))
    c2, l2 = ops.eval_summary(s.to(DEV), y.to(DEV), B, 0.5, segments_for(N))
    assert torch.equal(c1, c2) and _same(l1, l2)                      # two calls: identical bits


@pytest.mark.parametrize("C", [1, 10])
def test_misaligned_scores_one_bin_and_grids(C):
    N = 200_000
    s, y = make_case(C, N, 3)
    buf = torch.empty(N * C + 1, device=DEV)
    buf[1:] = s.reshape(-1).to(DEV)
    mis = buf[1:].view(N, C)
    assert mis.data_ptr() % 16 == 4
    segs = [70_000, 0, 1, 129_999]
    c1, l1 = ops.eval_summary(mis, y.to(DEV), 256, 0.5, segs)
    c2, l2 = reference.eval_summary(s, y, 256, 0.5, [0] + np.cumsum(segs).tolist())
    assert torch.equal(c1.cpu(), c2) and torch.allclose(l1.cpu(), l2, rtol=1e-6, atol=0)
    offs = torch.tensor([0] + np.cumsum(segs).tolist(), dtype=torch.int64)
    for grid in (1, 7, 132, 4096):
        c, l = _ext.require().eval_summary(mis, y.to(DEV), offs, 256, 0.5, grid)
        assert torch.equal(c, c1) and _same(l, l1)
    one = torch.full((N, C), 0.999 if C == 1 else -20.0)               # every row in one bin
    if C > 1:
        one[:, 0] = 20.0
    _check(one, y, 256, segs)


@pytest.mark.parametrize("C", [1, 10])
def test_a_hundred_segments_equal_a_hundred_launches(C):
    g = torch.Generator().manual_seed(9)
    segs = torch.randint(0, 5000, (100,), generator=g).tolist()
    segs[17] = 0
    s, y = make_case(C, sum(segs), 11)
    sd, yd = s.to(DEV), y.to(DEV)
    c, l = ops.eval_summary(sd, yd, 128, 0.5, segs)
    lo = 0
    for i, n in enumerate(segs):
        ci, li = ops.eval_summary(sd[lo:lo + n], yd[lo:lo + n], 128, 0.5)
        assert torch.equal(ci[0], c[i]) and _same(li[0], l[i])
        lo += n
    c2, l2 = reference.eval_summary(s, y, 128, 0.5, [0] + np.cumsum(segs).tolist())
    assert torch.equal(c.cpu(), c2) and torch.allclose(l.cpu(), l2, rtol=1e-6, atol=0)


@pytest.mark.parametrize("name", ["ffnn", "mlp"])
def test_model_summary_through_the_gpu_forward(name):
    from colearn_federated_learning_b200.fl.evaluate import forward_flat
    from colearn_federated_learning_b200.models import build_model, flatten_params
    torch.manual_seed(0)
    model = build_model(name).to(DEV)
    flat = flatten_params(model).to(DEV)
    x = torch.rand(10_000, 10, device=DEV)
    y = (torch.rand(10_000, device=DEV) > 0.5).float()
    got = fedeval.summarize(model, flat, x, y, 256, 0.5, [4000, 6000])
    out = forward_flat(model, flat, x).cpu()
    c, l = reference.eval_summary(out, y.cpu(), 256, 0.5, [0, 4000, 10000])
    for s, ci, li in zip(got, c, l):
        assert np.array_equal(s.counts, ci[2:].numpy()) and (s.n, s.n_invalid) == (int(ci[0]), int(ci[1]))
        assert s.loss_sum == pytest.approx(float(li), rel=1e-6)
        fedeval.check(s)
