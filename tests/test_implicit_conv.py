"""Implicit-GEMM convolution (csrc/conv_ops.cuh::ConvAddr, gemm_wgmma.cu conv modes).

The GPU-less evidence has two parts: (1) the *addressing* — the exact host+device decode the GEMM's producer warp runs
(``conv_kblock`` / ``conv_nblock``, called here through the host build) drives a Python model of tiled 4-D TMA boxes
(whole images, zero fill outside the tensor) and must reproduce conv2d / its input gradient / its weight gradient;
(2) the *definitions* of ``ops.conv.conv_gemm`` agree with autograd, and the trainer with the implicit schedule
agrees with the default one.  The sm_90a runs live in tests/test_gpu_schedules.py."""
import pytest
import torch
import torch.nn.functional as F

from colearn_federated_learning_b200.fl.convnet import ConvNetTrainer
from colearn_federated_learning_b200.models.registry import flatten_params
from colearn_federated_learning_b200.models.resnet import ResNet18
from colearn_federated_learning_b200.ops import conv

GEOMS = [  # (N, H, W, Cin, Cout)
    (4, 8, 8, 64, 64),      # layer1
    (8, 4, 4, 128, 128),    # layer2
    (32, 2, 2, 128, 64),    # layer3-like (2x2 images)
    (128, 1, 1, 64, 128),   # layer4-like (1x1 images: only the centre tap sees data)
]


def tma_box(x, c0, w0, h0, n0, box_n):
    """Model of a tiled 4-D TMA load of an NHWC tensor ``x [N, H, W, C]``: box (64, W, H, box_n) at signed coordinates
    (c0, w0, h0, n0), elements outside the tensor are zero; lines ordered w fastest, then h, then n."""
    n, h, w, c = x.shape
    out = torch.zeros(box_n, h, w, 64, dtype=x.dtype)
    for bi in range(box_n):
        ni = n0 + bi
        if not (0 <= ni < n):
            continue
        for hi in range(h):
            for wi in range(w):
                hh, ww = h0 + hi, w0 + wi
                if 0 <= hh < h and 0 <= ww < w:
                    out[bi, hi, wi] = x[ni, hh, ww, c0:c0 + 64]
    return out.view(box_n * h * w, 64)


def pack_w(wt):        # [Cout, Cin, 3, 3] -> [Cout, (kh, kw, c)]
    return wt.permute(0, 2, 3, 1).reshape(wt.shape[0], -1)


@pytest.mark.parametrize("n,h,w,cin,cout", GEOMS)
def test_producer_addressing_reproduces_the_three_conv_gemms(n, h, w, cin, cout):
    emul = conv.load_emulator()
    torch.manual_seed(n + h)
    x = torch.randn(n, h, w, cin, dtype=torch.float64)
    wt = torch.randn(cout, cin, 3, 3, dtype=torch.float64)
    x_nchw = x.permute(0, 3, 1, 2).clone().requires_grad_(True)
    wt_r = wt.clone().requires_grad_(True)
    z = F.conv2d(x_nchw, wt_r, padding=1)
    dz_nchw = torch.randn_like(z)
    z.backward(dz_nchw)
    z_ref = z.detach().permute(0, 2, 3, 1).reshape(n * h * w, cout)
    dx_ref = x_nchw.grad.permute(0, 2, 3, 1).reshape(n * h * w, cin)
    dw_ref = pack_w(wt_r.grad)
    dz = dz_nchw.permute(0, 2, 3, 1).contiguous()                       # NHWC [n, h, w, cout]
    wp = pack_w(wt)                                                     # [cout, 9*cin]
    m, hw = n * h * w, h * w

    # forward: A = x boxes of 128 pixels, B = packed weights K-major
    geom = [1, 0, cin, 3, 3, 1, hw, n, 0]
    got = torch.zeros(m, cout, dtype=torch.float64)
    for m0 in range(0, m, 128):
        for kb in range(9 * cin // 64):
            c0, w0, h0, n0, b_col, b_row = emul.conv_kblock(geom, kb, m0, 0)
            a = tma_box(x, c0, w0, h0, n0, 128 // hw)
            got[m0:m0 + 128] += a @ wp[b_row:b_row + cout, b_col:b_col + 64].t()
    torch.testing.assert_close(got, z_ref, rtol=1e-9, atol=1e-9)

    # dgrad: A = dz boxes (flipped taps), B = W^T [9*cin, cout] K-major, rows (tap, ci)
    wT = wp.t().contiguous()
    geom = [1, 1, cout, 3, 3, 1, hw, n, cin]
    got = torch.zeros(m, cin, dtype=torch.float64)
    for m0 in range(0, m, 128):
        for n0_ in range(0, cin, 64):                                    # two output-column tiles when cin = 128
            for kb in range(9 * cout // 64):
                c0, w0, h0, ni, b_col, b_row = emul.conv_kblock(geom, kb, m0, n0_)
                a = tma_box(dz, c0, w0, h0, ni, 128 // hw)
                got[m0:m0 + 128, n0_:n0_ + 64] += a @ wT[b_row:b_row + 64, b_col:b_col + 64].t()
    torch.testing.assert_close(got, dx_ref, rtol=1e-9, atol=1e-9)
    # ... and against the packed weights themselves (MN-major B): the same two numbers with swapped roles — b_col is the
    # ROW (co) of the [64 co x 64 ci] box, b_row its first COLUMN (tap*cin + n0)
    got = torch.zeros(m, cin, dtype=torch.float64)
    for m0 in range(0, m, 128):
        for n0_ in range(0, cin, 64):
            for kb in range(9 * cout // 64):
                c0, w0, h0, ni, b_col, b_row = emul.conv_kblock(geom, kb, m0, n0_)
                a = tma_box(dz, c0, w0, h0, ni, 128 // hw)
                got[m0:m0 + 128, n0_:n0_ + 64] += a @ wp[b_col:b_col + 64, b_row:b_row + 64]
    torch.testing.assert_close(got, dx_ref, rtol=1e-9, atol=1e-9)

    # wgrad: reduction over 64-pixel blocks; A = dz [pixels, cout], B = x boxes of 64 pixels per (tap, 64 channels)
    k_pad = (9 * cin + 127) // 128 * 128
    geom = [2, 0, cin, 3, 3, 1, hw, n, 0]
    dzm = dz.view(m, cout)
    got = torch.zeros(cout, k_pad, dtype=torch.float64)
    for kb in range(m // 64):
        a = dzm[kb * 64:(kb + 1) * 64]
        for blk in range(k_pad // 64):
            c0, w0, h0, ni = emul.conv_nblock(geom, blk, kb)
            b = tma_box(x, c0, w0, h0, ni, 64 // hw)
            got[:, blk * 64:(blk + 1) * 64] += a.t() @ b
    torch.testing.assert_close(got[:, :9 * cin], dw_ref, rtol=1e-9, atol=1e-9)
    assert float(got[:, 9 * cin:].abs().max() if k_pad > 9 * cin else 0.0) == 0.0   # the K padding stays exactly zero


@pytest.mark.parametrize("n,h,w,cin,cout", GEOMS[:3])
def test_conv_gemm_definitions_match_autograd(n, h, w, cin, cout):
    torch.manual_seed(1)
    x = torch.randn(n, cin, h, w)
    wt = torch.randn(cout, cin, 3, 3) * 0.1
    xr, wr = x.clone().requires_grad_(True), wt.clone().requires_grad_(True)
    z = F.conv2d(xr, wr, padding=1)
    dz4 = torch.randn_like(z)
    z.backward(dz4)
    m = n * h * w
    act = x.permute(0, 2, 3, 1).reshape(m, cin).contiguous()
    dz = dz4.permute(0, 2, 3, 1).reshape(m, cout).contiguous()
    cout_pad, k_pad = (cout + 127) // 128 * 128, (9 * cin + 127) // 128 * 128
    wp = torch.zeros(cout_pad, k_pad)
    wp[:cout, :9 * cin] = pack_w(wt)
    out = torch.zeros(m, cout_pad)
    conv.conv_gemm("fwd", act, wp, n, h, w, cin, 3, 3, 1, out_bf16=out)
    torch.testing.assert_close(out[:, :cout], z.detach().permute(0, 2, 3, 1).reshape(m, cout), rtol=1e-4, atol=1e-4)
    part = torch.zeros(3 * m * cout_pad)
    conv.conv_gemm("fwd", act, wp, n, h, w, cin, 3, 3, 1, split_k=3, split_out=part)
    torch.testing.assert_close(part.view(3, m, cout_pad).sum(0), out, rtol=1e-4, atol=1e-4)
    wT = wp[:cout].t().contiguous()                                      # [k_pad, cout]
    add = torch.randn(m, cin)
    dx = torch.zeros(m, cin)
    conv.conv_gemm("dgrad", dz, wT, n, h, w, cout, 3, 3, 1, out_bf16=dx, addend=add, rows_per_tap=cin)
    torch.testing.assert_close(dx, xr.grad.permute(0, 2, 3, 1).reshape(m, cin) + add, rtol=1e-4, atol=1e-4)
    dx2 = torch.zeros(m, cin)
    conv.conv_gemm("dgrad", dz, wp, n, h, w, cout, 3, 3, 1, out_bf16=dx2, addend=add, rows_per_tap=cin, w_packed=True)
    torch.testing.assert_close(dx2, dx, rtol=1e-5, atol=1e-5)
    master = wp.clone()
    conv.conv_gemm("wgrad", act, dz, n, h, w, cin, 3, 3, 1, m_pad=cout_pad, k_pad=k_pad, sgd_master=master, sgd_lr=0.5)
    part = torch.zeros(2 * cout_pad * k_pad + 100)                      # a larger shared scratch buffer is fine
    conv.conv_gemm("wgrad", act, dz, n, h, w, cin, 3, 3, 1, m_pad=cout_pad, k_pad=k_pad, split_k=2, split_out=part)
    torch.testing.assert_close(wp - 0.5 * part[: 2 * cout_pad * k_pad].view(2, cout_pad, k_pad).sum(0), master, rtol=1e-4, atol=1e-4)
    want = wp.clone()
    want[:cout, :9 * cin] -= 0.5 * pack_w(wr.grad)
    torch.testing.assert_close(master, want, rtol=1e-4, atol=1e-4)


@pytest.mark.usefixtures("legacy_conv_schedule")
@pytest.mark.parametrize("level,extra", [(1, {}), (2, {}), (2, {"split_k": 1, "dgrad_kn": False}),
                                         (2, {"split_k": 1, "dgrad_kn": True, "wgrad_mn": True})])
def test_implicit_schedule_is_the_same_step(level, extra):
    """``implicit=1``: forward and dgrad of the stride-1 3x3 convolutions read the activations through 4-D boxes (no
    im2col on the forward path, no dcol / col2im); ``implicit=2``: the wgrad too (no col at all).  Same products as
    the explicit schedule: the fp32-oracle step agrees to rounding."""
    torch.manual_seed(0)
    model = ResNet18(10)
    flat0 = flatten_params(model).clone()
    x, y = torch.randn(128, 3, 32, 32), torch.randint(0, 10, (128,))

    def run(dtype, **kw):
        flat = flat0.clone()
        tr = ConvNetTrainer(model, "cpu", 128, (32, 32), act_dtype=dtype, **kw)
        tr.load(flat, None)
        loss = float(tr.step(x, y, 0.05))
        tr.store(flat, None)
        return flat, loss, tr

    base, loss0, tr0 = run(torch.float32)
    got, loss1, tr1 = run(torch.float32, implicit=level, **extra)
    n_imp = sum(1 for cv in tr1.convs if cv.implicit)
    assert n_imp == 13 and not any(cv.implicit for cv in tr0.convs)
    assert abs(loss0 - loss1) < 1e-5
    # a different fp32 summation order in 13 layers of a random-init net: ~2e-4 of the update (both schedules sit 4e-3
    # away from autograd's update, see test_fp32_oracle_step_equals_autograd)
    assert float((got - base).norm() / (base - flat0).norm()) < 5e-4
    assert tr1.launches < tr0.launches
    b16, _, _ = run(torch.bfloat16)
    i16, _, _ = run(torch.bfloat16, implicit=level, **extra)
    d0, d1 = b16 - flat0, i16 - flat0
    # bf16 buffers: the implicit dgrad accumulates all taps in fp32 (no bf16 dcol in between), so the two schedules are
    # two different bf16 roundings of the same step — same class as bf16-vs-autocast in test_convnet_trainer (cos ~0.93)
    assert float((d0 * d1).sum() / (d0.norm() * d1.norm())) > 0.95
