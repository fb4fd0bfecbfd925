"""NHWC conv / BatchNorm / pooling ops (SURVEY K17).

Three layers of evidence, mirroring how the other kernels are tested (kernel vs a plain PyTorch fp32 reference):

1. the PyTorch *definitions* in ``ops/conv.py`` agree with ``torch.nn.functional`` + autograd (what the ops mean);
2. the *kernel bodies* (``csrc/conv_ops.cuh``) compiled for the host (``_colearn_emul``) agree with the definitions
   (``backend = "emul"``, runs on the CPU box);
3. the sm_90a kernels agree with the definitions (``backend = "cuda"``, ``@pytest.mark.gpu``).
"""
import contextlib

import pytest
import torch
import torch.nn.functional as F

from colearn_federated_learning_b200.ops import conv

BF = torch.bfloat16

BACKENDS = ["emul", pytest.param("cuda", marks=pytest.mark.gpu)]

# (N, C, H, W, K, stride, pad): the ResNet-18 geometries (small N) + odd sizes
GEOMS = [
    (2, 64, 8, 8, 3, 1, 1),      # layer1 3x3
    (2, 64, 8, 8, 3, 2, 1),      # layer2.0.conv1 (stride 2)
    (2, 64, 8, 8, 1, 2, 0),      # layer2.0.downsample (1x1 stride 2)
    (3, 128, 4, 4, 3, 1, 1),
    (2, 256, 2, 2, 3, 2, 1),     # -> 1x1
    (4, 512, 1, 1, 3, 1, 1),     # layer4: 1x1 spatial, only the centre tap sees data
    (2, 16, 9, 7, 3, 2, 1),      # odd, non-square
    (1, 8, 5, 6, 5, 1, 2),
]


@contextlib.contextmanager
def backend_ctx(backend):
    if backend == "emul":
        with conv.emulated():
            yield torch.device("cpu")
    elif backend == "simt":          # the CUDA launchers + kernels themselves on the CPU (csrc/host_shim.h)
        with conv.simt():
            yield torch.device("cpu")
    else:
        if not torch.cuda.is_available():
            pytest.skip("needs a GPU")
        yield torch.device("cuda:0")


def close(a, b, rtol=1.6e-2, atol=1e-3):
    torch.testing.assert_close(a.float().cpu(), b.float().cpu(), rtol=rtol, atol=atol)


def pad_to(n, m=128):
    return (n + m - 1) // m * m


# ---------------------------------------------------------------------------------------------------------------------
# 1. the definitions mean what torch means
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("geom", GEOMS)
def test_definitions_im2col_gemm_is_conv2d_and_col2im_is_its_adjoint(geom):
    n, c, h, w, k, s, p = geom
    torch.manual_seed(0)
    cout = 8
    x = torch.randn(n, c, h, w, requires_grad=True)
    wt = torch.randn(cout, c, k, k, requires_grad=True)
    oh, ow = conv.out_size(h, k, s, p), conv.out_size(w, k, s, p)
    kk = k * k * c
    col = torch.full((n * oh * ow, pad_to(kk)), 7.0)
    act = x.detach().permute(0, 2, 3, 1).reshape(n * h * w, c).contiguous()
    conv.im2col(conv.nhwc_view(act, n, h, w, c), col, k, k, s, p)
    assert col[:, kk:].abs().sum() == 0
    wp = wt.detach().permute(0, 2, 3, 1).reshape(cout, kk)                      # (kh, kw, c) packing
    z = col[:, :kk] @ wp.t()
    ref = F.conv2d(x, wt, stride=s, padding=p)
    close(z, ref.permute(0, 2, 3, 1).reshape(-1, cout), rtol=1e-4, atol=1e-4)
    # backward: dgrad through col2im, wgrad through col^T
    dz = torch.randn_like(z)
    ref.backward(dz.view(n, oh, ow, cout).permute(0, 3, 1, 2))
    dcol = torch.zeros_like(col)
    dcol[:, :kk] = dz @ wp
    dx = torch.zeros(n * h * w, c)
    conv.col2im(dcol, dx, None, n, h, w, c, k, k, s, p)
    close(dx, x.grad.permute(0, 2, 3, 1).reshape(-1, c), rtol=1e-4, atol=1e-4)
    dw = dz.t() @ col[:, :kk]
    close(dw, wt.grad.permute(0, 2, 3, 1).reshape(cout, kk), rtol=1e-4, atol=1e-4)


def test_definitions_batchnorm_matches_autograd():
    torch.manual_seed(1)
    m, c = 96, 64
    x = torch.randn(m, c, requires_grad=True) * 2 + 0.5
    x.retain_grad()
    res = torch.randn(m, c)
    gamma = (torch.rand(c) + 0.5).requires_grad_()
    beta = torch.randn(c).requires_grad_()
    rm, rv = torch.zeros(c), torch.ones(c)
    y = torch.relu(F.batch_norm(x, rm, rv, gamma, beta, True, 0.1, 1e-5) + res)
    dy = torch.randn(m, c)
    y.backward(dy)

    mean, invstd = torch.zeros(c), torch.zeros(c)
    rm2, rv2 = torch.zeros(c), torch.ones(c)
    partial = torch.zeros(conv.bn_partial_numel(m, c))
    xd = x.detach().contiguous()
    conv.bn_stats(xd, c, partial, mean, invstd, rm2, rv2, 1e-5, 0.1)
    close(rm2, rm, 1e-5, 1e-6)
    close(rv2, rv, 1e-5, 1e-6)
    out = torch.zeros(m, c)
    conv.bn_apply(xd, c, mean, invstd, gamma.detach(), beta.detach(), res, True, out)
    close(out, y, 1e-5, 1e-5)
    dg, db, dx, g = torch.zeros(c), torch.zeros(c), torch.zeros(m, c), torch.zeros(m, c)
    conv.bn_backward(xd, c, dy, out, mean, invstd, gamma.detach(), partial, dg, db, dx, g)
    close(dg, gamma.grad, 1e-4, 1e-4)
    close(db, beta.grad, 1e-4, 1e-4)
    close(dx, x.grad, 1e-4, 1e-5)
    close(g, dy * (y > 0), 0, 0)


def test_definitions_pooling_matches_autograd():
    torch.manual_seed(2)
    n, c, h, w = 2, 16, 9, 8
    x = torch.randn(n, c, h, w, requires_grad=True)
    y = F.max_pool2d(x, 3, 2, 1)
    oh, ow = y.shape[2:]
    dy = torch.randn_like(y)
    y.backward(dy)
    act = x.detach().permute(0, 2, 3, 1).reshape(-1, c).contiguous()
    out, idx = torch.zeros(n * oh * ow, c), torch.zeros(n * oh * ow, c, dtype=torch.uint8)
    conv.maxpool_fwd(act, out, idx, n, h, w, c, 3, 3, 2, 1)
    close(out, y.permute(0, 2, 3, 1).reshape(-1, c), 0, 0)
    dx = torch.zeros(n * h * w, c)
    conv.maxpool_bwd(dy.permute(0, 2, 3, 1).reshape(-1, c).contiguous(), idx, dx, n, h, w, c, 3, 3, 2, 1)
    close(dx, x.grad.permute(0, 2, 3, 1).reshape(-1, c), 0, 0)
    # global average pooling
    feat = torch.zeros(n, c)
    conv.avgpool_fwd(act, feat, n, h * w, c)
    close(feat, x.detach().mean((2, 3)), 1e-5, 1e-6)
    dxa = torch.zeros(n * h * w, c)
    conv.avgpool_bwd(feat, dxa, n, h * w, c)
    close(dxa.view(n, h * w, c), (feat / (h * w)).view(n, 1, c).expand(n, h * w, c), 1e-6, 1e-7)


# ---------------------------------------------------------------------------------------------------------------------
# 2./3. kernel bodies (host build) and sm_90a kernels against the definitions
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("backend", BACKENDS)
@pytest.mark.parametrize("geom", GEOMS)
def test_im2col_and_col2im_kernels(backend, geom):
    n, c, h, w, k, s, p = geom
    torch.manual_seed(3)
    oh, ow = conv.out_size(h, k, s, p), conv.out_size(w, k, s, p)
    kk, m = k * k * c, n * oh * ow
    act = torch.randn(n * h * w, c).to(BF)
    dcol = torch.randn(m, pad_to(kk)).to(BF)
    add = torch.randn(n * h * w, c).to(BF)
    col_ref = torch.full((m, pad_to(kk)), 7.0, dtype=BF)
    conv.im2col(conv.nhwc_view(act, n, h, w, c), col_ref, k, k, s, p)
    dx_ref, dx_ref2 = torch.zeros(n * h * w, c, dtype=BF), torch.zeros(n * h * w, c, dtype=BF)
    conv.col2im(dcol, dx_ref, add, n, h, w, c, k, k, s, p)
    conv.col2im(dcol, dx_ref2, None, n, h, w, c, k, k, s, p)
    with backend_ctx(backend) as dev:
        a = act.to(dev)
        col = torch.full((m, pad_to(kk)), 7.0, dtype=BF, device=dev)
        conv.im2col(conv.nhwc_view(a, n, h, w, c), col, k, k, s, p)
        assert torch.equal(col.cpu(), col_ref)                                   # a pure gather: bit exact
        dx = torch.zeros(n * h * w, c, dtype=BF, device=dev)
        conv.col2im(dcol.to(dev), dx, add.to(dev), n, h, w, c, k, k, s, p)
        close(dx, dx_ref, 1e-2, 2e-2)
        conv.col2im(dcol.to(dev), dx, None, n, h, w, c, k, k, s, p)
        close(dx, dx_ref2, 1e-2, 2e-2)


@pytest.mark.parametrize("backend", BACKENDS)
@pytest.mark.parametrize("src", ["nchw_f32", "nchw_bf16", "nhwc_c3"])
def test_im2col_stem_reads_the_user_batch_directly(backend, src):
    """7x7 / stride 2 / pad 3 on a 3-channel image: the scalar path (C % 8 != 0), strided fp32 or bf16 input."""
    torch.manual_seed(4)
    n, c, h, w, k, s, p = 2, 3, 32, 32, 7, 2, 3
    x = torch.randn(n, c, h, w)
    if src == "nchw_bf16":
        x = x.to(BF)
    elif src == "nhwc_c3":
        x = x.to(BF).permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2)      # NHWC storage, NCHW view
    oh = conv.out_size(h, k, s, p)
    kk = k * k * c
    ref = torch.full((n * oh * oh, pad_to(kk)), 7.0, dtype=BF)
    conv.im2col(x, ref, k, k, s, p)
    with backend_ctx(backend) as dev:
        col = torch.full((n * oh * oh, pad_to(kk)), 7.0, dtype=BF, device=dev)
        xd = x.to(dev)
        assert xd.stride() == x.stride()
        conv.im2col(xd, col, k, k, s, p)
        assert torch.equal(col.cpu(), ref)


@pytest.mark.parametrize("backend", BACKENDS)
@pytest.mark.parametrize("m,c,ldx", [(128, 64, 128), (8192, 64, 128), (2048, 128, 128), (512, 256, 256), (100, 64, 64), (4100, 512, 512)])
def test_batchnorm_kernels(backend, m, c, ldx):
    _batchnorm_case(backend, m, c, ldx, fused=False)


def _batchnorm_case(backend, m, c, ldx, fused):
    torch.manual_seed(5)
    x = (torch.randn(m, ldx) * 1.5 + 0.3).to(BF)
    res = torch.randn(m, c).to(BF)
    dy = torch.randn(m, c).to(BF)
    gamma, beta = torch.rand(c) + 0.5, torch.randn(c)

    counters = {}

    def run(dev, masked, with_res):
        xd = x.to(dev)
        mean, invstd = torch.zeros(c, device=dev), torch.zeros(c, device=dev)
        rm, rv = torch.zeros(c, device=dev), torch.ones(c, device=dev)
        partial = torch.zeros(conv.bn_partial_numel(m, c), device=dev)
        # single-launch reduction: the ticket counters are shared by all calls and must come back to zero each time
        cnt = counters.setdefault(str(dev), torch.zeros(c // 64, dtype=torch.int32, device=dev)) if fused else None
        conv.bn_stats(xd, c, partial, mean, invstd, rm, rv, 1e-5, 0.1, cnt)
        if fused:
            assert int(cnt.abs().sum()) == 0
        out = torch.zeros(m, c, dtype=BF, device=dev)
        conv.bn_apply(xd, c, mean, invstd, gamma.to(dev), beta.to(dev), res.to(dev) if with_res else None, masked, out)
        dg, db = torch.zeros(c, device=dev), torch.zeros(c, device=dev)
        dx, g = torch.zeros(m, c, dtype=BF, device=dev), torch.zeros(m, c, dtype=BF, device=dev)
        conv.bn_backward(xd, c, dy.to(dev), out if masked else None, mean, invstd, gamma.to(dev), partial, dg, db, dx,
                         g if masked else None, cnt)
        if fused:
            assert int(cnt.abs().sum()) == 0
        return [t.cpu() for t in (mean, invstd, rm, rv, out, dg, db, dx, g)]

    for masked, with_res in ((True, True), (False, False), (True, False)):
        ref = run(torch.device("cpu"), masked, with_res)
        with backend_ctx(backend) as dev:
            got = run(dev, masked, with_res)
        names = ["mean", "invstd", "running_mean", "running_var", "out", "dgamma", "dbeta", "dx", "g"]
        for name, a, b in zip(names, got, ref):
            if name in ("out", "dx", "g"):
                close(a, b, 1.6e-2, 2e-2)         # bf16 outputs: one ulp of slack
            elif name in ("dgamma", "dbeta"):
                close(a, b, 2e-3, 2e-3 * (m ** 0.5))
            else:
                close(a, b, 1e-4, 1e-5)


@pytest.mark.parametrize("backend", BACKENDS)
@pytest.mark.parametrize("geom", [(2, 64, 16, 16, 3, 2, 1), (2, 16, 9, 7, 3, 2, 1), (1, 8, 6, 6, 2, 2, 0)])
def test_pooling_kernels(backend, geom):
    n, c, h, w, k, s, p = geom
    torch.manual_seed(6)
    oh, ow = conv.out_size(h, k, s, p), conv.out_size(w, k, s, p)
    act = torch.relu(torch.randn(n * h * w, c)).to(BF)              # post-ReLU input: plenty of ties at 0
    dy = torch.randn(n * oh * ow, c).to(BF)
    out_ref, idx_ref = torch.zeros(n * oh * ow, c, dtype=BF), torch.zeros(n * oh * ow, c, dtype=torch.uint8)
    conv.maxpool_fwd(act, out_ref, idx_ref, n, h, w, c, k, k, s, p)
    dx_ref = torch.zeros(n * h * w, c, dtype=BF)
    conv.maxpool_bwd(dy, idx_ref, dx_ref, n, h, w, c, k, k, s, p)
    feat_ref, dxa_ref = torch.zeros(n, c, dtype=BF), torch.zeros(n * h * w, c, dtype=BF)
    conv.avgpool_fwd(act, feat_ref, n, h * w, c)
    conv.avgpool_bwd(feat_ref, dxa_ref, n, h * w, c)
    with backend_ctx(backend) as dev:
        out, idx = torch.zeros(n * oh * ow, c, dtype=BF, device=dev), torch.zeros(n * oh * ow, c, dtype=torch.uint8, device=dev)
        conv.maxpool_fwd(act.to(dev), out, idx, n, h, w, c, k, k, s, p)
        assert torch.equal(out.cpu(), out_ref) and torch.equal(idx.cpu(), idx_ref)
        dx = torch.zeros(n * h * w, c, dtype=BF, device=dev)
        conv.maxpool_bwd(dy.to(dev), idx, dx, n, h, w, c, k, k, s, p)
        close(dx, dx_ref, 1e-2, 1e-2)
        feat, dxa = torch.zeros(n, c, dtype=BF, device=dev), torch.zeros(n * h * w, c, dtype=BF, device=dev)
        conv.avgpool_fwd(act.to(dev), feat, n, h * w, c)
        close(feat, feat_ref, 1e-2, 1e-3)
        conv.avgpool_bwd(feat_ref.to(dev), dxa, n, h * w, c)
        close(dxa, dxa_ref, 1e-2, 1e-4)


@pytest.mark.parametrize("backend", BACKENDS)
def test_pack_and_unpack_params(backend):
    """arena ([Cout, Cin, KH, KW] + plain matrices) <-> padded, (kh, kw, c)-permuted GEMM layout, one launch."""
    torch.manual_seed(7)
    shapes = [(64, 3, 7, 7), (64, 64, 3, 3), (128, 64, 1, 1), (10, 512), (1, 64)]
    entries, off = [], 5
    for i, sh in enumerate(shapes):
        rows = sh[0]
        cols = int(torch.tensor(sh[1:]).prod())
        ch, khw = (sh[1], sh[2] * sh[3]) if len(sh) == 4 else (0, 1)
        rp = pad_to(rows) if rows > 1 else 1
        cp = pad_to(cols) if rows > 1 else cols
        entries.append(conv.PackEntry(f"p{i}", off, rows, cols, rp, cp, ch, khw))
        off += rows * cols + 3                                             # gaps: untouched arena elements
    arena = torch.randn(off + 4)

    def run(dev):
        plan = conv.PackPlan([conv.PackEntry(e.name, e.src_off, e.rows, e.cols, e.rows_pad, e.cols_pad, e.channels, e.khw)
                              for e in entries], dev)
        a = arena.to(dev)
        pf = torch.full((plan.total,), 9.0, device=dev)
        pb = torch.full((plan.total,), 9.0, device=dev, dtype=BF)
        conv.pack_params(a, pf, pb, plan)
        back = torch.full_like(a, -1.0)
        conv.pack_params(back, pf * 2, None, plan, unpack=True)
        return plan, pf.cpu(), pb.cpu(), back.cpu()

    plan, pf_ref, pb_ref, back_ref = run(torch.device("cpu"))
    # meaning: entry 1 is a 3x3 conv weight -> [Cout_pad, K_pad] with k = (kh, kw, c)
    e = plan.entries[1]
    wt = arena[e.src_off:e.src_off + 64 * 64 * 9].view(64, 64, 3, 3)
    assert torch.equal(plan.view(pf_ref, e)[:64, :576], wt.permute(0, 2, 3, 1).reshape(64, 576))
    assert plan.view(pf_ref, e)[64:].abs().max() == 0 and plan.view(pf_ref, e)[:, 576:].abs().max() == 0
    with backend_ctx(backend) as dev:
        _, pf, pb, back = run(dev)
    assert torch.equal(pf, pf_ref) and torch.equal(pb, pb_ref) and torch.equal(back, back_ref)
    touched = back_ref != -1.0
    assert torch.equal(back_ref[touched], (arena * 2)[touched]) and int(touched.sum()) == sum(e.rows * e.cols for e in entries)


@pytest.mark.parametrize("m,c,ldx", [(128, 64, 128), (8192, 64, 128), (512, 256, 256), (4100, 512, 512)])
def test_fused_batchnorm_reduction_kernel_bodies_on_host(m, c, ldx):
    """Single-launch BatchNorm reduction (the last block of a column group finalises, the ticket counter resets
    itself): the host build of the bodies against the definitions.  The sm_90a run lives in test_gpu_schedules."""
    _batchnorm_case("emul", m, c, ldx, fused=True)


# ---------------------------------------------------------------------------------------------------------------------
# split-K GEMM: partial accumulators + the reduction that applies the epilogue
# ---------------------------------------------------------------------------------------------------------------------
def test_splitk_reference_slices_add_up_to_the_plain_gemm():
    """``gemm_bf16(split_k=S)`` on the CPU defines the slice boundaries the kernel uses (k-blocks of 64, slice s =
    [nkb·s/S, nkb·(s+1)/S)); the slices must partition K for every S <= nkb, including S that do not divide nkb."""
    from colearn_federated_learning_b200 import ops
    torch.manual_seed(0)
    a, b = torch.randn(128, 64 * 7).to(BF), torch.randn(256, 64 * 7).to(BF)
    want = a.float() @ b.float().t()
    for s in (2, 3, 7):
        part = torch.full((s * 128 * 256 + 5,), 7.0)
        ops.gemm_bf16(a, b, split_k=s, split_out=part)
        torch.testing.assert_close(part[: s * 128 * 256].view(s, 128, 256).sum(0), want, rtol=1e-5, atol=1e-4)
        assert float(part[s * 128 * 256:].min()) == 7.0
    with pytest.raises(AssertionError):
        ops.gemm_bf16(a, b, split_k=8, split_out=torch.zeros(8 * 128 * 256))          # more slices than k-blocks
    with pytest.raises(AssertionError):
        ops.gemm_bf16(a, b, split_k=2, split_out=torch.zeros(2 * 128 * 256), out_f32=torch.zeros(128, 256))


@pytest.mark.parametrize("splits,rows,cols", [(2, 128, 128), (16, 128, 640), (64, 128, 256), (5, 4, 12)])
def test_splitk_reduce_kernel_body_on_host(splits, rows, cols):
    _splitk_reduce_case("emul", splits, rows, cols)


def _splitk_reduce_case(backend, splits, rows, cols):
    """Sum of the slices in slice order, then either the fused SGD step (fp32 master in place + bf16 shadow) or the
    bf16 output — bit-exact against the same expressions in PyTorch (fmaf for the SGD update)."""
    torch.manual_seed(splits)
    n = rows * cols
    part = torch.randn(splits, n)
    master0 = torch.randn(n)
    acc = part[0].clone()
    for s in range(1, splits):
        acc += part[s]
    lr = 0.05
    want_master = torch.addcmul(master0.double(), torch.tensor(-lr, dtype=torch.float32).double(), acc.double()).float()
    with backend_ctx(backend) as dev:
        p = torch.cat([part.reshape(-1), torch.full((8,), float("nan"))]).to(dev)     # slack must not be read
        master, shadow = master0.clone().to(dev), torch.zeros(n, dtype=BF, device=dev)
        conv.splitk_reduce(p, splits, n, master=master, lr=lr, shadow=shadow)
        out = torch.zeros(n + 4, dtype=BF, device=dev)
        conv.splitk_reduce(p, splits, n, out_bf16=out)
        only_master = master0.clone().to(dev)
        conv.splitk_reduce(p, splits, n, master=only_master, lr=lr)
    # fmaf(-lr, acc, w) rounds once: the double-precision product + sum rounded to fp32 is the same number
    torch.testing.assert_close(master.cpu(), want_master, rtol=0, atol=0)
    assert torch.equal(only_master.cpu(), master.cpu())
    assert torch.equal(shadow.cpu(), want_master.to(BF))
    assert torch.equal(out[:n].cpu(), acc.to(BF)) and float(out[n:].float().abs().max()) == 0
    # the definitions agree with the kernel bodies up to the non-fused multiply-add
    m2, s2 = master0.clone(), torch.zeros(n, dtype=BF)
    conv.splitk_reduce(part.reshape(-1).clone(), splits, n, master=m2, lr=lr, shadow=s2)
    torch.testing.assert_close(m2, want_master, rtol=1e-6, atol=1e-6)


def test_splitk_reduce_rejects_bad_arguments():
    with conv.emulated():
        p = torch.zeros(2 * 8)
        with pytest.raises(RuntimeError):
            conv.splitk_reduce(p, 2, 6, out_bf16=torch.zeros(6, dtype=BF))             # numel % 4
        with pytest.raises(RuntimeError):
            conv.splitk_reduce(p, 3, 8, out_bf16=torch.zeros(8, dtype=BF))             # part too small
        with pytest.raises(RuntimeError):
            conv.splitk_reduce(p, 2, 8, out_bf16=torch.zeros(4, dtype=BF))             # output too small


@pytest.mark.parametrize("m_units,n_tiles,num_kb,split,grid", [(1, 1, 512, 64, 148), (1, 5, 128, 16, 148), (32, 16, 16, 1, 148), (9, 7, 33, 5, 13),
                                                             (256, 1, 4, 1, 148), (3, 3, 7, 7, 4), (17, 2, 9, 2, 148)])
def test_gemm_work_decomposition_covers_every_tile_and_partitions_k(m_units, n_tiles, num_kb, split, grid):
    """The persistent GEMM's work list (the host build of ``work_to_tile`` / ``split_kb``, the functions every warp role
    of the kernel walks): over all CTAs each (tile, K slice) appears exactly once, the slices of a tile are disjoint,
    non-empty and cover all k-blocks, and the slices of one tile sit on consecutive CTAs (they run concurrently)."""
    emul = conv.load_emulator()
    seen = {}
    for cta in range(min(grid, m_units * n_tiles * split)):
        for mu, nb, ks, lo, hi in emul.gemm_work_list(cta, min(grid, m_units * n_tiles * split), m_units, n_tiles, num_kb, split):
            assert 0 <= mu < m_units and 0 <= nb < n_tiles and 0 <= ks < split and lo < hi
            assert (mu, nb, ks) not in seen
            seen[(mu, nb, ks)] = (lo, hi, cta)
    assert len(seen) == m_units * n_tiles * split
    for mu in range(m_units):
        for nb in range(n_tiles):
            ranges = [seen[(mu, nb, ks)][:2] for ks in range(split)]
            assert ranges[0][0] == 0 and ranges[-1][1] == num_kb
            assert all(ranges[i][1] == ranges[i + 1][0] for i in range(split - 1))
