"""sm_90a kernel numerics vs the plain-PyTorch fp32 reference of the same op (needs a GPU)."""
import pytest
import torch

from colearn_federated_learning_b200 import ops
from colearn_federated_learning_b200.models import FFNN, MLP, TestingRemote, flatten_params
from colearn_federated_learning_b200.ops import reference as R

pytestmark = pytest.mark.gpu


def _dev():
    return torch.device("cuda", 0)


def test_extension_loaded():
    from colearn_federated_learning_b200.ops import _ext
    assert _ext.require() is not None
    assert _ext.so_path() is not None


@pytest.mark.parametrize("ctor,loss", [(FFNN, "bce"), (FFNN, "sse"), (MLP, "xent"), (TestingRemote, "sse"), (TestingRemote, "mse")])
@pytest.mark.parametrize("bsz,n,epochs,max_b", [(1, 97, 1, -1), (1, 200, 2, 150), (8, 203, 2, -1), (32, 64, 3, 5)])
@pytest.mark.parametrize("variant", [5, 6, 3, 1])
def test_persistent_mlp_matches_reference(ctor, loss, bsz, n, epochs, max_b, variant):
    torch.manual_seed(0)
    model = ctor()
    spec = model.spec
    flat0 = flatten_params(model).clone()
    x = torch.rand(n, spec.dims[0])
    if loss == "xent":
        y = torch.randint(0, spec.dims[-1], (n, 1)).float()
    else:
        y = (torch.rand(n, spec.dims[-1]) > 0.5).float()
    perm = R.make_permutation(n, epochs, seed=5)
    ref = flat0.clone()
    ref_last = R.mlp_local_sgd(ref, spec.dims, x, y, perm, bsz, 0.05, epochs, max_b, loss, spec.out_activation)
    got = flat0.clone().to(_dev())
    last = ops.mlp_local_sgd(got, spec.dims, x.to(_dev()), y.to(_dev()), perm.to(_dev()), bsz, 0.05, epochs, max_b,
                             loss, spec.out_activation, variant=variant)
    torch.cuda.synchronize()
    assert torch.allclose(got.cpu(), ref, atol=2e-4, rtol=2e-3), (got.cpu() - ref).abs().max()
    assert torch.allclose(last.cpu(), ref_last, atol=1e-3, rtol=1e-2)


def test_persistent_mlp_multi_client_scale_and_delta():
    torch.manual_seed(1)
    model = MLP()
    spec = model.spec
    dev = _dev()
    theta = flatten_params(model).clone().to(dev)
    k, n = 5, 64
    xs = [torch.rand(n, 10, device=dev) for _ in range(k)]
    ys = [torch.randint(0, 2, (n, 1), device=dev).float() for _ in range(k)]
    perm = R.make_permutation(n, 1, 9).to(dev)
    slots = torch.zeros(k, theta.numel(), device=dev)
    losses = torch.zeros(k, 2, device=dev)
    w = [0.1, 0.2, 0.3, 0.15, 0.25]
    tasks = [ops.ClientTask(x=xs[i], y=ys[i], theta_in=theta, theta_out=slots[i], perm=perm, loss_out=losses[i],
                            out_scale=w[i], delta_mode=(i % 2 == 1)) for i in range(k)]
    descs = ops.build_client_descs(tasks, dev)
    ops.mlp_local_sgd_multi(spec.dims, spec.out_activation, descs, k, batch_size=1, lr=0.05, loss="xent")
    torch.cuda.synchronize()
    for i in range(k):
        ref = theta.cpu().clone()
        R.mlp_local_sgd(ref, spec.dims, xs[i].cpu(), ys[i].cpu(), perm.cpu(), 1, 0.05, 1, -1, "xent")
        want = w[i] * (ref - theta.cpu()) if i % 2 == 1 else w[i] * ref
        assert torch.allclose(slots[i].cpu(), want, atol=2e-4, rtol=2e-3)


@pytest.mark.parametrize("ctor,loss", [(MLP, "xent"), (FFNN, "sse")])
@pytest.mark.parametrize("variant", [5, 6, 3, 1])
def test_in_kernel_shuffle_equals_the_tabulated_permutation(variant, ctor, loss):
    """ClientDesc::perm_seed: the gather of the persistent kernel computes the keyed Feistel order itself — same bits as
    training through the table feistel_perm_kernel writes for that seed (rows perm_row0 .. perm_row0 + epochs - 1), and the
    host implementation of the bijection agrees with the device one."""
    torch.manual_seed(4)
    dev = _dev()
    model = ctor()
    spec = model.spec
    theta = flatten_params(model).clone().to(dev)
    n, epochs, seed, row0 = 333, 3, 987654321, 5
    x, y = torch.rand(n, 10, device=dev), torch.randint(0, 2, (n, 1), device=dev).float()
    table = ops.device_permutation(n, row0 + epochs, seed, dev)
    host = ops._ext.require().feistel_permutation(n, row0 + epochs, seed, torch.device("cpu"))
    assert torch.equal(table.cpu(), host)
    outs = []
    scratch = torch.empty(epochs * n, dtype=torch.int32, device=dev)
    for kw in (dict(perm=table[row0:].contiguous()), dict(perm_seed=seed, perm_row0=row0, perm_scratch=scratch)):
        out, lo = torch.zeros_like(theta), torch.zeros(2, device=dev)
        descs = ops.build_client_descs([ops.ClientTask(x=x, y=y, theta_in=theta, theta_out=out, loss_out=lo, **kw)], dev)
        ops.mlp_local_sgd_multi(spec.dims, spec.out_activation, descs, 1, batch_size=1, lr=0.05, epochs=epochs, loss=loss, variant=variant)
        torch.cuda.synchronize()
        outs.append((out.clone(), lo.clone()))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
    assert not torch.equal(outs[0][0], theta)
    if variant != 1 and ctor is MLP:        # (v1 and the 4-layer nets' index ring compute the order inside the gather: no table)
        assert torch.equal(scratch.view(epochs, n), table[row0:])


def test_mlp_forward():
    torch.manual_seed(2)
    for ctor in (FFNN, MLP, TestingRemote):
        m = ctor()
        flat = flatten_params(m).to(_dev())
        x = torch.rand(300, m.spec.dims[0])
        out = ops.mlp_forward(flat, m.spec.dims, x.to(_dev()), m.spec.out_activation)
        assert torch.allclose(out.cpu(), m(x).detach(), atol=1e-5, rtol=1e-4)


def test_sgd_and_fedavg():
    dev = _dev()
    torch.manual_seed(3)
    for n in (5, 4994, 1 << 20, (1 << 20) + 3):
        p, g = torch.randn(n, device=dev), torch.randn(n, device=dev)
        want = p - 0.01 * g
        ops.sgd_step(p, g, 0.01)
        assert torch.allclose(p, want, atol=1e-6)
    models = torch.randn(8, 4994, device=dev)
    w = torch.rand(8, device=dev)
    w = w / w.sum()
    assert torch.allclose(ops.fedavg_flat(models, w), R.fedavg_flat(models, w), atol=1e-5)
    theta = torch.randn(4994, device=dev)
    want = R.fedavg_apply(theta.clone(), models, w, 0.7)
    ops.fedavg_apply(theta, models, w, 0.7)
    assert torch.allclose(theta, want, atol=1e-5)


def test_losses():
    dev = _dev()
    torch.manual_seed(4)
    z, y = torch.randn(1000, 1, device=dev) * 3, (torch.rand(1000, 1, device=dev) > 0.5).float()
    l, dz = ops.sigmoid_bce(z, y)
    rl, rdz = R.sigmoid_bce(z.cpu(), y.cpu())
    assert torch.allclose(l.cpu(), rl, atol=1e-5) and torch.allclose(dz.cpu(), rdz, atol=1e-6)
    out = torch.randn(500, 3, device=dev)
    tgt = torch.randn(500, 3, device=dev)
    l, d = ops.sse_loss(out, tgt)
    assert torch.allclose(l.cpu(), ((out - tgt) ** 2).sum().cpu(), rtol=1e-5)
    assert torch.allclose(d, 2 * (out - tgt), atol=1e-6)
    for cols in (2, 10, 100):
        logits = torch.randn(777, cols, device=dev) * 2
        labels = torch.randint(0, cols, (777,), device=dev)
        l, d = ops.softmax_xent(logits, labels)
        rl, rd = R.softmax_xent(logits.cpu(), labels.cpu())
        assert torch.allclose(l.cpu(), rl, atol=1e-5, rtol=1e-5)
        assert torch.allclose(d.cpu(), rd, atol=1e-6)
        lb, db = ops.softmax_xent(logits.to(torch.bfloat16), labels, bf16_grad=True)
        assert db.dtype == torch.bfloat16 and abs(lb.item() - rl.item()) < 0.05
    # one-block loss head on padded operands (both GEMM-shaped trainers): bf16 gradient in place, bias gradient, loss
    from colearn_federated_learning_b200.ops import conv as C
    for rows, cols, ld in ((128, 10, 64), (1024, 2, 64), (5, 100, 128), (333, 128, 128)):
        big = torch.randn(rows + 3, ld, device=dev) * 2
        lab = torch.randint(0, cols, (rows + 3,), device=dev)
        dz = torch.full((rows + 3, ld), 7.0, dtype=torch.bfloat16, device=dev)
        dbias = torch.full((ld,), 7.0, device=dev)
        outs = []
        for _ in range(2):
            loss = C.softmax_xent_head(big, lab, rows, cols, dl_bf16=dz, db=dbias)
            outs.append((loss.clone(), dz.clone(), dbias.clone()))
        assert all(torch.equal(a, b) for a, b in zip(outs[0], outs[1]))                 # fixed summation order
        rl, rdl = R.softmax_xent(big[:rows, :cols].cpu(), lab[:rows].cpu())
        assert torch.allclose(loss.cpu(), rl, atol=1e-5, rtol=1e-5)
        assert torch.allclose(dz[:rows, :cols].float().cpu(), rdl, atol=1e-6, rtol=1e-2)
        assert torch.allclose(dbias[:cols].cpu(), rdl.sum(0), atol=1e-6, rtol=1e-4)
        assert bool((dz[rows:] == 7).all()) and bool((dz[:, cols:] == 7).all()) and bool((dbias[cols:] == 7).all())


def test_eval_argmax_minmax_perm_convert():
    dev = _dev()
    torch.manual_seed(5)
    p = torch.rand(999, device=dev).clamp(1e-4, 1 - 1e-4)
    y = (torch.rand(999, device=dev) > 0.5).float()
    l, c = ops.eval_binary(p, y)
    rl, rc = R.eval_binary(p.cpu(), y.cpu())
    assert torch.allclose(l.cpu(), rl, rtol=1e-5) and int(c) == int(rc)
    x = torch.randn(257, 10, device=dev)
    assert torch.equal(ops.argmax_rows(x).cpu(), x.cpu().argmax(1, keepdim=True))
    s = ops.minmax_scale(x)
    assert torch.allclose(s.min(0).values, torch.zeros(10, device=dev), atol=1e-6)
    assert torch.allclose(s.max(0).values, torch.ones(10, device=dev), atol=1e-6)
    for n in (1, 2, 7, 1000, 4099):
        pm = ops.device_permutation(n, 3, seed=11, device=dev).cpu()
        for r in range(3):
            assert sorted(pm[r].tolist()) == list(range(n))
        if n > 100:
            assert not torch.equal(pm[0], pm[1])
    v = torch.randn(1003, device=dev)
    assert torch.equal(ops.fp32_to_bf16(v), v.to(torch.bfloat16))


@pytest.mark.parametrize("m,n,k,tile_n,cluster", [(128, 128, 64, 0, 0), (256, 384, 512, 0, 0), (1024, 4096, 4096, 0, 0),
                                                  (128, 256, 128, 256, 1), (384, 512, 320, 256, 1), (1024, 4096, 4096, 128, 0),
                                                  (256, 256, 64, 256, 2), (512, 768, 448, 256, 2), (2048, 4096, 1024, 256, 2),
                                                  (1024, 4096, 4096, 256, 1),
                                                  (256, 256, 64, 256, 3), (512, 768, 448, 256, 3), (1024, 4096, 4096, 256, 3),
                                                  # the ResNet-18 conv shapes (fl/convnet.py): stem fwd / wgrad, layer1 dgrad / wgrad
                                                  (32768, 128, 256, 0, 0), (128, 256, 32768, 0, 0), (8192, 640, 64, 0, 0),
                                                  (128, 640, 8192, 0, 0), (128, 4608, 128, 0, 0)])
def test_gemm_tcgen05_plain(m, n, k, tile_n, cluster):
    dev = _dev()
    torch.manual_seed(6)
    a = (torch.randn(m, k, device=dev) * 0.5).to(torch.bfloat16)
    b = (torch.randn(n, k, device=dev) * 0.5).to(torch.bfloat16)
    out = torch.empty(m, n, device=dev, dtype=torch.float32)
    ops.gemm_bf16(a, b, out_f32=out, tile_n=tile_n, cluster=cluster)
    torch.cuda.synchronize()
    ref = a.float() @ b.float().t()
    err = (out - ref).abs().max().item()
    assert err < 1e-2 * max(1.0, ref.abs().max().item()), err


@pytest.mark.parametrize("cluster", [0, 3])
def test_gemm_tcgen05_epilogues(cluster):
    dev = _dev()
    torch.manual_seed(7)
    m, n, k = 256, 256, 192
    a = (torch.randn(m, k, device=dev) * 0.3).to(torch.bfloat16)
    b = (torch.randn(n, k, device=dev) * 0.3).to(torch.bfloat16)
    bias = torch.randn(n, device=dev)
    ref = a.float() @ b.float().t()
    # bias + relu, bf16 + transposed outputs
    o, ot = torch.empty(m, n, device=dev, dtype=torch.bfloat16), torch.empty(n, m, device=dev, dtype=torch.bfloat16)
    ops.gemm_bf16(a, b, bias=bias, relu=True, out_bf16=o, out_bf16_t=ot, cluster=cluster)
    want = torch.relu(ref + bias)
    assert torch.allclose(o.float(), want, atol=5e-2, rtol=2e-2)
    assert torch.equal(ot, o.t().contiguous())
    # relu mask (dgrad) + column sums (bias grad)
    mask = (torch.randn(m, n, device=dev)).to(torch.bfloat16)
    of = torch.empty(m, n, device=dev)
    cs = torch.zeros(m // 32, n, device=dev)
    ops.gemm_bf16(a, b, relu_mask=mask, out_f32=of, colsum=cs, cluster=cluster)
    assert torch.allclose(of, ref * (mask.float() > 0), atol=1e-2, rtol=1e-2)
    want_cs = (ref * (mask.float() > 0)).view(m // 32, 32, n).sum(1)                      # per-32-row-block partials
    assert torch.allclose(cs, want_cs, atol=5e-2, rtol=1e-2)
    bias_t = torch.randn(n - 3, device=dev)
    before = bias_t.clone()
    g = ops.bias_sgd_from_partials(bias_t, cs, 0.1)
    assert torch.allclose(g, want_cs.sum(0), atol=5e-2, rtol=1e-2) and torch.allclose(bias_t, before - 0.1 * g[: n - 3], atol=1e-5)
    # fused SGD on the fp32 master + shadow refresh
    master = torch.randn(m, n, device=dev)
    want_master = master - 0.1 * ref
    sh, sht = torch.empty(m, n, device=dev, dtype=torch.bfloat16), torch.empty(n, m, device=dev, dtype=torch.bfloat16)
    ops.gemm_bf16(a, b, sgd_master=master, sgd_lr=0.1, sgd_shadow=sh, sgd_shadow_t=sht, cluster=cluster)
    assert torch.allclose(master, want_master, atol=1e-2, rtol=1e-2)
    assert torch.equal(sh, master.to(torch.bfloat16)) and torch.equal(sht, master.t().contiguous().to(torch.bfloat16))


def test_layerwise_tcgen05_trainer_matches_autograd():
    """Wide-MLP local SGD on wgmma GEMMs (fwd / dgrad / wgrad + fused SGD) vs fp32 autograd."""
    from colearn_federated_learning_b200.fl import FitConfig
    from colearn_federated_learning_b200.fl.layerwise import LayerwiseMLPTrainer
    from colearn_federated_learning_b200.models import MLPNet, MLPSpec
    dev = _dev()
    torch.manual_seed(0)
    spec = MLPSpec((10, 256, 256, 2), "none", "xent")
    m = MLPNet(spec)
    flat = flatten_params(m).clone().to(dev)
    x, y = torch.rand(384, 10), torch.randint(0, 2, (384, 1)).float()
    cfg = FitConfig(model="x", loss="xent", batch_size=128, lr=0.1)
    assert LayerwiseMLPTrainer.supports(spec, cfg)
    tr = LayerwiseMLPTrainer(spec, flat, 128, dgrad_kn=False, wgrad_mn=False)   # K-major form (W^T copies kept); the default
    last = tr.fit(flat, x.to(dev), y.to(dev), cfg, None)                         # in-place operand form: test_gpu_schedules.py
    torch.cuda.synchronize()
    opt = torch.optim.SGD(m.parameters(), lr=0.1)
    for lo in (0, 128, 256):
        opt.zero_grad()
        l = torch.nn.functional.cross_entropy(m(x[lo:lo + 128]), y[lo:lo + 128].view(-1).long())
        l.backward()
        opt.step()
    ref = flatten_params(m)
    assert abs(float(last) - float(l)) < 2e-2
    assert (flat.cpu() - ref).abs().max() < 5e-3, (flat.cpu() - ref).abs().max()
    # shadows are consistent with the fp32 master after the fused-SGD epilogue
    tr.sync_transposes()          # W^T is refreshed on demand (by the next dgrad): bring it up to date before looking at it
    w2 = flat[spec.offsets()[1][0]: spec.offsets()[1][0] + 256 * 256].view(256, 256)
    assert torch.equal(tr.Ws[1], w2.to(torch.bfloat16)) and torch.equal(tr.WsT[1], w2.t().contiguous().to(torch.bfloat16))


def test_transpose_bf16():
    dev = _dev()
    x = torch.randn(300, 70, device=dev).to(torch.bfloat16)
    assert torch.equal(ops.transpose_bf16(x), x.t().contiguous())


def test_smpc_ring_kernels_match_cpu():
    """SURVEY K18: int64 ring ops on CUDA cores (fix-precision encode/decode, wrap-around matmul, Beaver matmul)."""
    from colearn_federated_learning_b200.smpc import CryptoProvider, fix_precision, float_precision, share
    from colearn_federated_learning_b200.smpc.sharing import ring_matmul
    dev = _dev()
    torch.manual_seed(8)
    x = torch.randn(37, 19) * 5
    assert torch.equal(fix_precision(x.to(dev)).cpu(), fix_precision(x))
    assert torch.allclose(float_precision(fix_precision(x.to(dev))).cpu(), float_precision(fix_precision(x)))
    a = torch.randint(-(2 ** 62), 2 ** 62, (33, 21), dtype=torch.int64)
    b = torch.randint(-(2 ** 62), 2 ** 62, (21, 18), dtype=torch.int64)
    assert torch.equal(ring_matmul(a.to(dev), b.to(dev)).cpu(), ring_matmul(a, b))      # exact, incl. wrap-around
    p = CryptoProvider(4)
    u, v = torch.randn(6, 9), torch.randn(9, 5)
    su, sv = share(fix_precision(u.to(dev)), p), share(fix_precision(v.to(dev)), p)
    got = float_precision(su.matmul(sv).truncate().get()).cpu()
    assert (got - u @ v).abs().max() < 0.03
