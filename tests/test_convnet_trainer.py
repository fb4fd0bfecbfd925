"""ResNet-18 local training on the repo's own ops (fl/convnet.py, SURVEY K17) against autograd."""
import contextlib

import pytest
import torch
import torch.nn.functional as F

from colearn_federated_learning_b200.fl.convnet import ConvNetTrainer
from colearn_federated_learning_b200.fl.trainer import FitConfig, local_fit
from colearn_federated_learning_b200.models.registry import flatten_params, param_layout, unflatten_params
from colearn_federated_learning_b200.models.resnet import ResNet18
from colearn_federated_learning_b200.ops import conv

B = 128


def autograd_step(flat0, x, y, lr, autocast=False):
    ref = ResNet18(10)
    unflatten_params(ref, flat0)
    ref.train()
    with torch.autocast("cpu", dtype=torch.bfloat16, enabled=autocast):
        out = ref(x)
    loss = F.cross_entropy(out.float(), y)
    loss.backward()
    with torch.no_grad():
        for p in ref.parameters():
            p.sub_(lr * p.grad)
    return flatten_params(ref), float(loss), ref


def cosines(model, d_a, d_b):
    out = {}
    for name, _, off, n in param_layout(model):
        a, b = d_a[off:off + n], d_b[off:off + n]
        out[name] = float((a * b).sum() / (a.norm() * b.norm() + 1e-30))
    return out


def test_fp32_oracle_step_equals_autograd():
    """With fp32 buffers the PyTorch definitions of the ops make the trainer an exact re-implementation of
    forward + backward + SGD: every parameter update must match autograd's, and so must the BatchNorm buffers."""
    torch.manual_seed(0)
    model = ResNet18(10)
    flat0 = flatten_params(model).clone()
    x, y = torch.randn(B, 3, 32, 32), torch.randint(0, 10, (B,))
    flat_ref, loss_ref, ref = autograd_step(flat0, x, y, 0.05)
    flat = flat0.clone()
    tr = ConvNetTrainer(model, "cpu", B, (32, 32), act_dtype=torch.float32)
    tr.load(flat, model)
    loss = float(tr.step(x, y, 0.05))
    tr.store(flat, model)
    assert abs(loss - loss_ref) < 1e-4
    cs = cosines(model, flat - flat0, flat_ref - flat0)
    assert min(cs.values()) > 0.9999, min(cs.items(), key=lambda kv: kv[1])
    rel = float((flat - flat_ref).norm() / (flat_ref - flat0).norm())
    assert rel < 2e-2, rel
    mods, rmods = dict(model.named_modules()), dict(ref.named_modules())
    for name, m in mods.items():
        if hasattr(m, "running_mean"):
            torch.testing.assert_close(m.running_mean, rmods[name].running_mean, rtol=1e-4, atol=1e-5)
            torch.testing.assert_close(m.running_var, rmods[name].running_var, rtol=1e-4, atol=1e-5)
            assert int(m.num_batches_tracked) == 1


@pytest.mark.usefixtures("legacy_conv_schedule")
@pytest.mark.parametrize("level", [1, 2])
def test_split_k_schedule_is_the_same_step(level):
    """Split-K (wgrads of the stem / layer1 / layer2 cut over pixel slices, level 2: the layer4 forwards too) only
    changes the fp32 summation order: in fp32-oracle mode the step must agree with the un-split step to rounding,
    and with bf16 buffers through the host build of the kernel bodies it must stay in the same class."""
    torch.manual_seed(0)
    model = ResNet18(10)
    flat0 = flatten_params(model).clone()
    x, y = torch.randn(B, 3, 32, 32), torch.randint(0, 10, (B,))

    def run(split, dtype, emul=False):
        flat = flat0.clone()
        tr = ConvNetTrainer(model, "cpu", B, (32, 32), act_dtype=dtype, split_k=split)
        with (conv.emulated() if emul else contextlib.nullcontext()):
            tr.load(flat, None)
            loss = float(tr.step(x, y, 0.05))
            tr.store(flat, None)
        return flat, loss, tr

    base, loss0, tr0 = run(0, torch.float32)
    got, loss1, tr1 = run(level, torch.float32)
    assert all(cv.s_wgrad == 1 and cv.s_fwd == 1 for cv in tr0.convs)
    assert tr1.stem.s_wgrad == 64 and tr1.blocks[0].c1.s_wgrad == 16 and tr1.blocks[2].c1.s_wgrad == 4
    assert (max(cv.s_fwd for cv in tr1.convs) > 1) == (level == 2)
    assert tr1.launches > tr0.launches                      # one reduction launch per split GEMM
    assert abs(loss0 - loss1) < 1e-4
    rel = float((got - base).norm() / (base - flat0).norm())
    assert rel < 1e-4, rel
    # bf16 buffers, host build of the kernel bodies (splitk_reduce_body): same class as the un-split bf16 step
    b16, _, _ = run(0, torch.bfloat16, emul=True)
    s16, _, _ = run(level, torch.bfloat16, emul=True)
    d0, d1 = b16 - flat0, s16 - flat0
    assert float((d0 * d1).sum() / (d0.norm() * d1.norm())) > (0.999 if level == 1 else 0.95)


@pytest.mark.usefixtures("legacy_conv_schedule")
@pytest.mark.parametrize("split", [0, 1])
def test_mn_major_wgrad_schedule_is_the_same_step(split):
    """``wgrad_mn``: the wgrad GEMMs read ``dz`` / ``col`` in place (reduction over rows) instead of transposed copies —
    the same products, so the fp32-oracle step must agree with the default schedule to rounding; fewer launches."""
    torch.manual_seed(0)
    model = ResNet18(10)
    flat0 = flatten_params(model).clone()
    x, y = torch.randn(B, 3, 32, 32), torch.randint(0, 10, (B,))

    def run(mn, dtype, kn=False):
        flat = flat0.clone()
        tr = ConvNetTrainer(model, "cpu", B, (32, 32), act_dtype=dtype, split_k=split, wgrad_mn=mn, dgrad_kn=kn)
        tr.load(flat, None)
        loss = float(tr.step(x, y, 0.05))
        tr.store(flat, None)
        return flat, loss, tr.launches

    base, loss0, n0 = run(False, torch.float32)
    got, loss1, n1 = run(True, torch.float32)
    assert n0 - n1 == 2 * 20                                 # two transposes per convolution are gone
    # ... and with the dgrads reading the packed weights in place, the W^T copies (load + refresh per step) too
    got_kn, loss2, n2 = run(True, torch.float32, kn=True)
    assert n1 - n2 == 2 * 20 and abs(loss0 - loss2) < 1e-5
    assert float((got_kn - base).norm() / (base - flat0).norm()) < 1e-4
    assert abs(loss0 - loss1) < 1e-5
    assert float((got - base).norm() / (base - flat0).norm()) < 1e-4
    b16, _, _ = run(False, torch.bfloat16)
    m16, _, _ = run(True, torch.bfloat16)
    d0, d1 = b16 - flat0, m16 - flat0
    assert float((d0 * d1).sum() / (d0.norm() * d1.norm())) > 0.9999


def test_mn_major_gemm_reference_definition():
    """``gemm_bf16(a[K, a_cols], b[K, N], mn_m=M)`` = ``aᵀ·b`` zero-extended to M rows, with every epilogue of the
    K-major form (here: fused SGD + both shadows, and split-K partials)."""
    from colearn_federated_learning_b200 import ops
    torch.manual_seed(1)
    a, b = torch.randn(256, 64).to(torch.bfloat16), torch.randn(256, 384).to(torch.bfloat16)
    want = torch.zeros(128, 384)
    want[:64] = a.float().t() @ b.float()
    out = torch.empty(128, 384)
    ops.gemm_bf16(a, b, mn_m=128, out_f32=out)
    torch.testing.assert_close(out, want, rtol=1e-5, atol=1e-4)
    master, shadow, shadow_t = torch.ones(128, 384), torch.zeros(128, 384, dtype=torch.bfloat16), torch.zeros(384, 128, dtype=torch.bfloat16)
    ops.gemm_bf16(a, b, mn_m=128, sgd_master=master, sgd_lr=0.5, sgd_shadow=shadow, sgd_shadow_t=shadow_t)
    torch.testing.assert_close(master, 1 - 0.5 * want, rtol=1e-5, atol=1e-4)
    assert torch.equal(shadow, master.to(torch.bfloat16)) and torch.equal(shadow_t, shadow.t())
    part = torch.zeros(4 * 128 * 384)
    ops.gemm_bf16(a, b, mn_m=128, split_k=4, split_out=part)
    torch.testing.assert_close(part.view(4, 128, 384).sum(0), want, rtol=1e-5, atol=1e-4)
    torch.testing.assert_close(part.view(4, 128, 384)[1, :64], a[64:128].float().t() @ b[64:128].float(), rtol=1e-5, atol=1e-4)
    with pytest.raises(AssertionError):
        ops.gemm_bf16(a, b, mn_m=64, out_f32=out)            # M must be a multiple of 128


def test_pick_split_heuristic():
    pick = ConvNetTrainer._pick_split
    assert pick(128, 256, 32768) == 64          # stem wgrad: 1 tile of 128x256, 512 k-blocks -> 64 slices of 8
    assert pick(128, 640, 8192) == 16           # layer1 wgrad: 5 tiles of 128x128, 128 k-blocks
    assert pick(128, 640, 8192, min_slices=32) == 1
    assert pick(32768, 128, 256) == 1           # plenty of tiles
    assert pick(128, 128, 64) == 1              # nothing to split
    for m, n, k in [(128, 256, 32768), (128, 640, 8192), (128, 1152, 2048), (128, 512, 4608)]:
        s = pick(m, n, k)
        assert s == 1 or (k // 64) // s >= 8    # every slice keeps a pipeline's worth of k-blocks


@pytest.mark.parametrize("mode", ["fp32", "definitions", "emulated"])
def test_eval_mode_inference_matches_module_eval(mode):
    """``infer``: eval-mode forward (running statistics) in chunks of 128 with a zero-padded last chunk."""
    torch.manual_seed(3)
    model = ResNet18(10)
    with torch.no_grad():                                 # non-trivial running statistics
        for m in model.modules():
            if hasattr(m, "running_mean"):
                m.running_mean.normal_(0, 0.2)
                m.running_var.uniform_(0.5, 1.5)
    x = torch.randn(B + 37, 3, 32, 32)
    model.eval()
    with torch.no_grad():
        want = model(x)
    flat = flatten_params(model).clone()
    tr = ConvNetTrainer(model, "cpu", B, (32, 32), act_dtype=torch.float32 if mode == "fp32" else torch.bfloat16)
    with (conv.emulated() if mode == "emulated" else contextlib.nullcontext()):
        tr.load(flat, model)
        got = tr.infer(x)
    assert got.shape == want.shape
    if mode == "fp32":
        torch.testing.assert_close(got, want, rtol=1e-3, atol=1e-3)
    else:
        assert float((got - want).abs().max()) < 0.15 * float(want.abs().max()) + 0.05
        assert float((got.argmax(1) == want.argmax(1)).float().mean()) > 0.9


@pytest.mark.parametrize("mode", ["definitions", "emulated"])
def test_bf16_step_is_as_close_to_fp32_autograd_as_autocast_is(mode):
    """bf16 activations on a random-init ResNet-18 with 1x1 final feature maps are noisy (torch's own autocast path
    only reaches cos ~0.93 against fp32); the bf16 trainer — through the PyTorch definitions and through the host
    build of the kernel bodies — must be in the same class, and must agree with autocast at least as well."""
    torch.manual_seed(0)
    model = ResNet18(10)
    flat0 = flatten_params(model).clone()
    x, y = torch.randn(B, 3, 32, 32), torch.randint(0, 10, (B,))
    flat_ref, loss_ref, _ = autograd_step(flat0, x, y, 0.05)
    flat_ac, _, _ = autograd_step(flat0, x, y, 0.05, autocast=True)
    flat = flat0.clone()
    tr = ConvNetTrainer(model, "cpu", B, (32, 32))
    with (conv.emulated() if mode == "emulated" else contextlib.nullcontext()):
        tr.load(flat, None)
        loss = float(tr.step(x, y, 0.05))
        tr.store(flat, None)
    assert abs(loss - loss_ref) < 2e-2
    d, d_ref, d_ac = flat - flat0, flat_ref - flat0, flat_ac - flat0
    cos = lambda a, b: float((a * b).sum() / (a.norm() * b.norm()))  # noqa: E731
    assert cos(d, d_ref) > cos(d_ac, d_ref) - 0.03
    assert cos(d, d_ref) > 0.9 and cos(d, d_ac) > 0.9
    cs = cosines(model, d, d_ref)
    assert cs["fc.weight"] > 0.995 and cs["layer4.1.conv2.weight"] > 0.97


def test_local_fit_native_conv_path_on_cpu(monkeypatch):
    """``COLEARN_CONV_PATH=native`` routes ResNet-18 through the trainer (several steps, shuffled, in place on the
    arena) and the result tracks the autograd path; a ragged last batch falls back to autograd."""
    torch.manual_seed(1)
    model = ResNet18(10)
    flat0 = flatten_params(model).clone()
    x, y = torch.randn(2 * B, 3, 32, 32), torch.randint(0, 10, (2 * B,))
    cfg = FitConfig(model="resnet18", loss="xent", batch_size=B, epochs=1, lr=0.02, shuffle=True, seed=3)
    monkeypatch.setenv("COLEARN_CONV_PATH", "native")
    flat = flat0.clone()
    loss, path = local_fit(flat, model, x, y, cfg)
    assert path == "convnet" and torch.isfinite(loss)
    monkeypatch.setenv("COLEARN_CONV_PATH", "torch")
    flat_t = flat0.clone()
    loss_t, path_t = local_fit(flat_t, ResNet18(10), x, y, cfg)
    assert path_t == "torch"
    d, d_t = flat - flat0, flat_t - flat0
    # two bf16 steps against two fp32 steps of a chaotic random-init net: same direction, not the same digits
    assert float((d * d_t).sum() / (d.norm() * d_t.norm())) > 0.6
    assert abs(float(loss) - float(loss_t)) < 0.3
    monkeypatch.setenv("COLEARN_CONV_PATH", "native")
    _, path_r = local_fit(flat0.clone(), model, x[: B + 5], y[: B + 5], cfg)
    assert path_r == "torch"


@pytest.mark.gpu
def test_gpu_step_matches_definitions_and_autocast():
    """The sm_90a path (im2col / BatchNorm / pooling kernels + wgmma GEMMs) against the CPU definitions of the
    same ops on the same data, layer by layer on the forward, and against fp32 autograd on the update."""
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    torch.manual_seed(0)
    dev = torch.device("cuda:0")
    model = ResNet18(10)
    flat0 = flatten_params(model).clone()
    x, y = torch.randn(B, 3, 32, 32), torch.randint(0, 10, (B,))
    flat_ref, loss_ref, _ = autograd_step(flat0, x, y, 0.05)
    cpu = ConvNetTrainer(model, "cpu", B, (32, 32))
    fc = flat0.clone()
    cpu.load(fc, None)
    loss_cpu = float(cpu.step(x, y, 0.05))
    cpu.store(fc, None)
    gpu = ConvNetTrainer(model, dev, B, (32, 32))
    fg = flat0.to(dev)
    gpu.load(fg, None)
    torch.testing.assert_close(gpu.mpk.cpu(), cpu_mpk0(model, flat0), rtol=0, atol=0)
    loss_gpu = float(gpu.step(x.to(dev), y.to(dev), 0.05))
    gpu.store(fg, None)
    torch.cuda.synchronize()
    # the stem sees identical inputs on both sides: bit-exact gather, GEMM and statistics within rounding
    assert torch.equal(gpu.stem.col.cpu(), cpu.stem.col)
    torch.testing.assert_close(gpu.stem.z.float().cpu(), cpu.stem.z.float(), rtol=2e-2, atol=2e-2)
    torch.testing.assert_close(gpu.stem.mean.cpu(), cpu.stem.mean, rtol=1e-3, atol=1e-3)
    torch.testing.assert_close(gpu.stem.out.float().cpu(), cpu.stem.out.float(), rtol=3e-2, atol=3e-2)
    assert abs(loss_gpu - loss_ref) < 2e-2 and abs(loss_gpu - loss_cpu) < 2e-2
    d, d_ref, d_cpu = fg.cpu() - flat0, flat_ref - flat0, fc - flat0
    cos = lambda a, b: float((a * b).sum() / (a.norm() * b.norm()))  # noqa: E731
    assert cos(d, d_ref) > 0.9 and cos(d, d_cpu) > 0.9
    cs = cosines(model, d, d_ref)
    assert cs["fc.weight"] > 0.995 and cs["layer4.1.conv2.weight"] > 0.97
    assert torch.isfinite(fg).all()


def cpu_mpk0(model, flat0):
    tr = ConvNetTrainer(model, "cpu", B, (32, 32))
    tr.load(flat0.clone(), None)
    return tr.mpk


@pytest.mark.gpu
def test_gpu_fit_reduces_loss_and_matches_torch_path(monkeypatch):
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    torch.manual_seed(2)
    dev = torch.device("cuda:0")
    model = ResNet18(10).to(dev)
    flat = flatten_params(model)
    # a learnable toy problem: the label is the sign pattern of the channel means
    x = torch.randn(4 * B, 3, 32, 32, device=dev)
    y = ((x.mean((2, 3)) > 0).long() * torch.tensor([1, 2, 4], device=dev)).sum(1)
    cfg = FitConfig(model="resnet18", loss="xent", batch_size=B, epochs=3, lr=0.05, shuffle=True, seed=1)
    monkeypatch.setenv("COLEARN_CONV_PATH", "native")
    first = None
    for r in range(3):
        loss, path = local_fit(flat, model, x, y, cfg, round_idx=r)
        assert path == "convnet"
        first = float(loss) if first is None else first
    assert float(loss) < first and torch.isfinite(flat).all()
