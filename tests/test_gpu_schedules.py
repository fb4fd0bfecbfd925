"""GPU tests of the ResNet-18 step schedules, the GEMM operand / scheduling modes behind them (split-K, MN-major operands,
implicit-GEMM convolution, programmatic dependent launch) and the engine modes added in round 2.  Every re-scheduling is
compared with the round-1 schedule (fixture ``legacy_conv_schedule``: all of fl.convnet.SCHEDULE_DEFAULTS at 0); the
shipped defaults — the fastest measured combination — are the "all switches" rows of these tests plus
tests/test_convnet_trainer.py."""
import os

import pytest
import torch

from colearn_federated_learning_b200.fl.convnet import ConvNetTrainer
from colearn_federated_learning_b200.fl.evaluate import evaluate, predict
from colearn_federated_learning_b200.models.registry import flatten_params
from colearn_federated_learning_b200.models.resnet import ResNet18

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures("legacy_conv_schedule")]


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda:0")


def test_resnet_eval_mode_inference_on_own_kernels():
    dev = _dev()
    torch.manual_seed(3)
    model = ResNet18(10)
    with torch.no_grad():
        for m in model.modules():
            if hasattr(m, "running_mean"):
                m.running_mean.normal_(0, 0.2)
                m.running_var.uniform_(0.5, 1.5)
    x = torch.randn(128 + 37, 3, 32, 32)
    model.eval()
    with torch.no_grad():
        want = model(x)
    model.to(dev)
    flat = flatten_params(model)
    tr = ConvNetTrainer.cached(model, flat, 128, (32, 32))
    tr.load(flat, model)
    got = tr.infer(x.to(dev)).cpu()
    assert float((got - want).abs().max()) < 0.15 * float(want.abs().max()) + 0.05
    assert float((got.argmax(1) == want.argmax(1)).float().mean()) > 0.9
    # public helpers route conv nets on a GPU through the same path
    pred = predict(model, x.to(dev), flat).cpu().view(-1)
    assert float((pred == want.argmax(1)).float().mean()) > 0.9
    res = evaluate(model, x.to(dev), want.argmax(1).to(dev), flat, verbose=False)
    assert res["accuracy"] > 0.9 and res["n"] == x.shape[0]


@pytest.mark.parametrize("m,c,ldx", [(128, 64, 128), (8192, 64, 128), (512, 256, 256), (4100, 512, 512)])
def test_fused_batchnorm_reduction_kernel(m, c, ldx):
    """``bn_reduce_finalize_kernel`` (ticket counter, last block finalises) against the two-kernel definitions."""
    _dev()
    from test_conv_ops import _batchnorm_case
    _batchnorm_case("cuda", m, c, ldx, fused=True)


@pytest.mark.parametrize("flags", [{"COLEARN_CONV_STREAMS": "1"}, {"COLEARN_CONV_SHADOW_T": "1"}, {"COLEARN_CONV_FUSED_BN": "1"},
                                   {"COLEARN_CONV_STREAMS": "1", "COLEARN_CONV_SHADOW_T": "1", "COLEARN_CONV_FUSED_BN": "1"}])
def test_optional_step_optimisations_do_not_change_the_result(flags, monkeypatch):
    """Second stream for the wgrad chains / W^T from the wgrad epilogue / single-launch BatchNorm reductions are
    re-schedulings of the same kernels on the same data: the parameters after two steps (one eager, one through the
    CUDA graph) must match the default schedule (bitwise for the stream and W^T variants)."""
    dev = _dev()
    torch.manual_seed(0)
    x = torch.randn(256, 3, 32, 32, device=dev)
    y = torch.randint(0, 10, (256,), device=dev)

    def run():
        torch.manual_seed(1)
        model = ResNet18(10).to(dev)
        flat = flatten_params(model)
        tr = ConvNetTrainer(model, dev, 128, (32, 32))
        tr.load(flat, model)
        for lo in (0, 128):
            tr._graph_step(x[lo:lo + 128], y[lo:lo + 128], 0.05)
        tr.store(flat, model)
        torch.cuda.synchronize()
        return flat.clone()

    for k in ("COLEARN_CONV_STREAMS", "COLEARN_CONV_SHADOW_T", "COLEARN_CONV_FUSED_BN"):
        monkeypatch.delenv(k, raising=False)
    base = run()
    for k, v in flags.items():
        monkeypatch.setenv(k, v)
    got = run()
    if "COLEARN_CONV_FUSED_BN" in flags:
        torch.testing.assert_close(got, base, rtol=1e-2, atol=1e-3)
    else:
        assert torch.equal(got, base)


@pytest.mark.parametrize("splits,rows,cols", [(2, 128, 128), (16, 128, 640), (64, 128, 256), (5, 4, 12)])
def test_splitk_reduce_kernel(splits, rows, cols):
    _dev()
    from test_conv_ops import _splitk_reduce_case
    _splitk_reduce_case("cuda", splits, rows, cols)


@pytest.mark.parametrize("m,n,k,s,tile_n", [(128, 256, 32768, 64, 0), (128, 640, 8192, 16, 0), (256, 128, 4096, 3, 0),
                                            (512, 512, 1024, 4, 128), (128, 512, 4608, 9, 256), (1024, 256, 512, 8, 0)])
def test_gemm_split_k_partials(m, n, k, s, tile_n):
    """Split-K mode of the 1-CTA wgmma GEMM: every slice's raw accumulator against the fp32 product of the same
    K range (slice boundaries = the CPU definition's), their sum against the un-split kernel, untouched slack."""
    dev = _dev()
    from colearn_federated_learning_b200 import ops
    torch.manual_seed(m + n + s)
    a = torch.randn(m, k, device=dev).to(torch.bfloat16)
    b = torch.randn(n, k, device=dev).to(torch.bfloat16)
    part = torch.full((s * m * n + 64,), 7.0, device=dev)
    ops.gemm_bf16(a, b, split_k=s, split_out=part, tile_n=tile_n)
    plain = torch.empty(m, n, device=dev)
    ops.gemm_bf16(a, b, out_f32=plain)
    torch.cuda.synchronize()
    assert float(part[s * m * n:].min()) == 7.0 and float(part[s * m * n:].max()) == 7.0
    want = torch.zeros(s * m * n + 64)
    ops.gemm_bf16(a.cpu(), b.cpu(), split_k=s, split_out=want)
    got = part[: s * m * n].view(s, m, n).cpu()
    torch.testing.assert_close(got, want[: s * m * n].view(s, m, n), rtol=2e-3, atol=2e-2 * (k / s / 512) ** 0.5)
    torch.testing.assert_close(got.sum(0), plain.cpu(), rtol=2e-3, atol=5e-2)
    # and through the reduction: the bf16 result of the un-split kernel
    out = torch.empty(m, n, device=dev, dtype=torch.bfloat16)
    ref = torch.empty(m, n, device=dev, dtype=torch.bfloat16)
    from colearn_federated_learning_b200.ops import conv as C
    C.splitk_reduce(part, s, m * n, out_bf16=out)
    ops.gemm_bf16(a, b, out_bf16=ref)
    torch.testing.assert_close(out.float().cpu(), ref.float().cpu(), rtol=1.6e-2, atol=0.5)


def _one_step_update(dev, graph: bool):
    """Parameter update of ONE ResNet-18 step (eager, or the first replay of the step graph) from a fixed initial state."""
    torch.manual_seed(0)
    x = torch.randn(128, 3, 32, 32, device=dev)
    y = torch.randint(0, 10, (128,), device=dev)
    torch.manual_seed(1)
    model = ResNet18(10).to(dev)
    flat = flatten_params(model)
    flat0 = flat.clone()
    tr = ConvNetTrainer(model, dev, 128, (32, 32))
    tr.load(flat, model)
    (tr._graph_step if graph else tr.step)(x, y, 0.05)
    tr.store(flat, model)
    torch.cuda.synchronize()
    return flat.clone() - flat0


def _assert_same_step(got, base, cos_min=0.9995):
    """One step apart, two schedules differ by fp32 summation order / bf16 rounding only.  (TWO steps are no test: at this
    learning rate a 1e-6 relative perturbation of the parameters after step 1 already moves the 2-step update to cosine
    0.982 under the SAME schedule — so a 2-step comparison measures chaos, not kernels.)"""
    cos = float((got * base).sum() / (got.norm() * base.norm()))
    rel = float((got - base).norm() / base.norm())
    assert torch.isfinite(got).all() and cos > cos_min and rel < 0.03, (cos, rel)


@pytest.mark.parametrize("graph", [False, True])
@pytest.mark.parametrize("level", ["1", "2"])
def test_split_k_step_matches_default_schedule(level, graph, monkeypatch):
    """COLEARN_CONV_SPLITK: the split only changes the fp32 summation order of the affected GEMMs."""
    dev = _dev()
    base = _one_step_update(dev, graph)
    monkeypatch.setenv("COLEARN_CONV_SPLITK", level)
    _assert_same_step(_one_step_update(dev, graph), base)


def _mn_case(dev, kdim, a_cols, m, n, split=0):
    from colearn_federated_learning_b200 import ops
    torch.manual_seed(kdim + n)
    a = torch.randn(kdim, a_cols, device=dev).to(torch.bfloat16)
    b = torch.randn(kdim, n, device=dev).to(torch.bfloat16)
    want = torch.zeros(m, n)
    want[:a_cols] = a.float().cpu().t() @ b.float().cpu()
    tol = dict(rtol=2e-3, atol=2e-2 * (kdim / 512) ** 0.5)
    if split:
        part = torch.full((split * m * n + 64,), 7.0, device=dev)
        ops.gemm_bf16(a, b, mn_m=m, split_k=split, split_out=part)
        torch.cuda.synchronize()
        assert float(part[split * m * n:].min()) == 7.0
        got = part[: split * m * n].view(split, m, n).sum(0).cpu()
    else:
        out = torch.full((m, n), 7.0, device=dev)
        ops.gemm_bf16(a, b, mn_m=m, out_f32=out)
        torch.cuda.synchronize()
        got = out.cpu()
    return got, want, tol


@pytest.mark.parametrize("kdim,a_cols,m,n,split", [(64, 128, 128, 128, 0), (128, 64, 128, 128, 0), (8192, 64, 128, 640, 0),
                                                   (32768, 64, 128, 256, 64), (512, 256, 256, 2304, 0), (128, 512, 512, 4608, 0),
                                                   (8192, 64, 128, 640, 16), (2048, 128, 128, 1152, 4)])
def test_gemm_mn_major_operands(kdim, a_cols, m, n, split):
    """C = AᵀB with A [K, a_cols], B [K, N] row-major (MN-major wgmma descriptors, boxes of 64 rows x 64 columns; the
    rows of C past a_cols are TMA zero fill) against the fp32 product."""
    got, want, tol = _mn_case(_dev(), kdim, a_cols, m, n, split)
    torch.testing.assert_close(got, want, **tol)


@pytest.mark.parametrize("m,kdim,b_rows,n", [(128, 64, 64, 128), (8192, 64, 128, 640), (2048, 128, 128, 1152), (512, 256, 256, 2304),
                                             (128, 512, 512, 4608), (32768, 64, 128, 256)])
def test_gemm_mn_major_b_operand(m, kdim, b_rows, n):
    """C = A·B[:K] with A [M, K] K-major and B [b_rows >= K, N] row-major (MN-major B descriptor): the conv dgrad
    against the packed weights."""
    dev = _dev()
    from colearn_federated_learning_b200 import ops
    torch.manual_seed(m + n)
    a = torch.randn(m, kdim, device=dev).to(torch.bfloat16)
    b = torch.randn(b_rows, n, device=dev).to(torch.bfloat16)
    out = torch.full((m, n), 7.0, device=dev, dtype=torch.bfloat16)
    ops.gemm_bf16(a, b, b_kn=True, out_bf16=out)
    torch.cuda.synchronize()
    want = a.float() @ b[:kdim].float()
    torch.testing.assert_close(out.float(), want, rtol=1.6e-2, atol=2e-2 * (kdim / 64) ** 0.5)


def test_gemm_mn_major_fused_sgd_epilogue():
    dev = _dev()
    from colearn_federated_learning_b200 import ops
    torch.manual_seed(5)
    a = torch.randn(2048, 128, device=dev).to(torch.bfloat16)
    b = torch.randn(2048, 1152, device=dev).to(torch.bfloat16)
    master = torch.randn(128, 1152, device=dev)
    m0 = master.clone()
    shadow = torch.zeros(128, 1152, device=dev, dtype=torch.bfloat16)
    shadow_t = torch.zeros(1152, 128, device=dev, dtype=torch.bfloat16)
    ops.gemm_bf16(a, b, mn_m=128, sgd_master=master, sgd_lr=0.01, sgd_shadow=shadow, sgd_shadow_t=shadow_t)
    torch.cuda.synchronize()
    want = m0 - 0.01 * (a.float().t() @ b.float())
    torch.testing.assert_close(master, want, rtol=1e-3, atol=1e-2)
    assert torch.equal(shadow, master.to(torch.bfloat16)) and torch.equal(shadow_t, shadow.t().contiguous())


@pytest.mark.parametrize("flags", [{"COLEARN_CONV_WGRAD_MN": "1"}, {"COLEARN_CONV_DGRAD_KN": "1"},
                                   {"COLEARN_CONV_WGRAD_MN": "1", "COLEARN_CONV_SPLITK": "1"},
                                   {"COLEARN_CONV_WGRAD_MN": "1", "COLEARN_CONV_DGRAD_KN": "1", "COLEARN_CONV_SPLITK": "1",
                                    "COLEARN_CONV_FUSED_BN": "1"},
                                   {"COLEARN_CONV_WGRAD_MN": "1", "COLEARN_CONV_DGRAD_KN": "1", "COLEARN_CONV_SPLITK": "2",
                                    "COLEARN_CONV_STREAMS": "1", "COLEARN_CONV_FUSED_BN": "1"}])
def test_mn_major_wgrad_step_matches_default_schedule(flags, monkeypatch):
    dev = _dev()
    graph = "COLEARN_CONV_STREAMS" in flags            # the second stream only exists inside the captured step
    base = _one_step_update(dev, graph)
    for k, v in flags.items():
        monkeypatch.setenv(k, v)
    _assert_same_step(_one_step_update(dev, graph), base)


# ---- implicit-GEMM convolution (4-D TMA boxes): tests/test_implicit_conv.py has the host-side evidence -----------------
IMPLICIT_GEOMS = [(128, 8, 8, 64, 64), (128, 4, 4, 128, 128), (128, 2, 2, 256, 256), (128, 1, 1, 512, 512), (128, 4, 4, 64, 128)]


def _implicit_case(n, h, w, cin, cout):
    import torch.nn.functional as F
    torch.manual_seed(n + h + cin)
    x = torch.randn(n, cin, h, w).to(torch.bfloat16)
    wt = (torch.randn(cout, cin, 3, 3) * (2.0 / (9 * cin)) ** 0.5).to(torch.bfloat16)
    xr, wr = x.float().requires_grad_(True), wt.float().requires_grad_(True)
    z = F.conv2d(xr, wr, padding=1)
    dz4 = torch.randn_like(z).to(torch.bfloat16)
    z.backward(dz4.float())
    m = n * h * w
    nhwc = lambda t, c: t.permute(0, 2, 3, 1).reshape(m, c).contiguous()      # noqa: E731
    cout_pad, k_pad = (cout + 127) // 128 * 128, (9 * cin + 127) // 128 * 128
    wp = torch.zeros(cout_pad, k_pad, dtype=torch.bfloat16)
    wp[:cout, :9 * cin] = wt.permute(0, 2, 3, 1).reshape(cout, -1)
    return dict(m=m, act=nhwc(x, cin), dz=nhwc(dz4, cout), wp=wp, cout_pad=cout_pad, k_pad=k_pad,
                z=nhwc(z.detach(), cout), dx=nhwc(xr.grad, cin), dw=wr.grad.permute(0, 2, 3, 1).reshape(cout, -1))


@pytest.mark.parametrize("n,h,w,cin,cout", IMPLICIT_GEOMS)
def test_implicit_conv_forward_and_dgrad(n, h, w, cin, cout):
    dev = _dev()
    from colearn_federated_learning_b200.ops import conv as C
    d = _implicit_case(n, h, w, cin, cout)
    m = d["m"]
    out = torch.full((m, d["cout_pad"]), 7.0, device=dev, dtype=torch.bfloat16)
    C.conv_gemm("fwd", d["act"].to(dev), d["wp"].to(dev), n, h, w, cin, 3, 3, 1, out_bf16=out)
    torch.cuda.synchronize()
    torch.testing.assert_close(out[:, :cout].float().cpu(), d["z"], rtol=2e-2, atol=3e-2)
    assert float(out[:, cout:].float().abs().max() if d["cout_pad"] > cout else 0.0) == 0.0
    # split-K over the (tap, channel-block) loop
    s = 3
    part = torch.zeros(s * m * d["cout_pad"], device=dev)
    C.conv_gemm("fwd", d["act"].to(dev), d["wp"].to(dev), n, h, w, cin, 3, 3, 1, split_k=s, split_out=part)
    torch.cuda.synchronize()
    torch.testing.assert_close(part.view(s, m, d["cout_pad"]).sum(0)[:, :cout].cpu(), d["z"], rtol=2e-2, atol=3e-2)
    # dgrad (+ residual gradient); cin = 64 exercises the 128x64 tile
    wT = d["wp"][:cout].t().contiguous().to(dev)
    add = torch.randn(m, cin).to(torch.bfloat16)
    dx = torch.full((m, cin), 7.0, device=dev, dtype=torch.bfloat16)
    C.conv_gemm("dgrad", d["dz"].to(dev), wT, n, h, w, cout, 3, 3, 1, out_bf16=dx, addend=add.to(dev), rows_per_tap=cin)
    torch.cuda.synchronize()
    torch.testing.assert_close(dx.float().cpu(), d["dx"] + add.float(), rtol=2e-2, atol=5e-2)


@pytest.mark.parametrize("n,h,w,cin,cout", IMPLICIT_GEOMS)
def test_implicit_conv_dgrad_packed_weights(n, h, w, cin, cout):
    """The implicit dgrad against the packed weights themselves (MN-major B operand, no W^T copy)."""
    dev = _dev()
    from colearn_federated_learning_b200.ops import conv as C
    d = _implicit_case(n, h, w, cin, cout)
    m = d["m"]
    add = torch.randn(m, cin).to(torch.bfloat16)
    dx2 = torch.full((m, cin), 7.0, device=dev, dtype=torch.bfloat16)
    C.conv_gemm("dgrad", d["dz"].to(dev), d["wp"].to(dev), n, h, w, cout, 3, 3, 1, out_bf16=dx2, addend=add.to(dev), rows_per_tap=cin,
                w_packed=True)
    torch.cuda.synchronize()
    torch.testing.assert_close(dx2.float().cpu(), d["dx"] + add.float(), rtol=2e-2, atol=5e-2)


@pytest.mark.parametrize("n,h,w,cin,cout", IMPLICIT_GEOMS)
def test_implicit_conv_wgrad(n, h, w, cin, cout):
    dev = _dev()
    from colearn_federated_learning_b200.ops import conv as C
    d = _implicit_case(n, h, w, cin, cout)
    cp, kp = d["cout_pad"], d["k_pad"]
    master = torch.zeros(cp, kp, device=dev)
    shadow = torch.zeros(cp, kp, device=dev, dtype=torch.bfloat16)
    C.conv_gemm("wgrad", d["act"].to(dev), d["dz"].to(dev), n, h, w, cin, 3, 3, 1, m_pad=cp, k_pad=kp, sgd_master=master,
                sgd_lr=-1.0, sgd_shadow=shadow)                                  # lr = -1: master = +dW
    torch.cuda.synchronize()
    scale = float(d["dw"].abs().max())
    torch.testing.assert_close(master[:cout, :9 * cin].cpu(), d["dw"], rtol=2e-2, atol=2e-2 * scale)
    assert float(master[cout:].abs().max() if cp > cout else 0.0) == 0.0 and float(master[:, 9 * cin:].abs().max() if kp > 9 * cin else 0.0) == 0.0
    assert torch.equal(shadow, master.to(torch.bfloat16))
    s = min(4, (n * h * w) // 64)          # the reduction runs over the pixels: at least one 64-pixel k-block per split
    part = torch.zeros(s * cp * kp + 64, device=dev)
    C.conv_gemm("wgrad", d["act"].to(dev), d["dz"].to(dev), n, h, w, cin, 3, 3, 1, m_pad=cp, k_pad=kp, split_k=s, split_out=part)
    torch.cuda.synchronize()
    torch.testing.assert_close(part[: s * cp * kp].view(s, cp, kp).sum(0), master, rtol=1e-3, atol=1e-3 * scale)


@pytest.mark.parametrize("flags", [{"COLEARN_CONV_IMPLICIT": "1"}, {"COLEARN_CONV_IMPLICIT": "2"},
                                   {"COLEARN_CONV_IMPLICIT": "2", "COLEARN_CONV_WGRAD_MN": "1", "COLEARN_CONV_DGRAD_KN": "1",
                                    "COLEARN_CONV_SPLITK": "1", "COLEARN_CONV_FUSED_BN": "1"},
                                   {"COLEARN_CONV_IMPLICIT": "2", "COLEARN_CONV_WGRAD_MN": "1", "COLEARN_CONV_DGRAD_KN": "1",
                                    "COLEARN_CONV_SPLITK": "1", "COLEARN_CONV_FUSED_BN": "1", "COLEARN_CONV_STREAMS": "1"}])   # = SCHEDULE_DEFAULTS
def test_implicit_step_matches_default_schedule(flags, monkeypatch):
    dev = _dev()
    base = _one_step_update(dev, True)
    for k, v in flags.items():
        monkeypatch.setenv(k, v)
    _assert_same_step(_one_step_update(dev, True), base, cos_min=0.999)


# ---- programmatic dependent launch (default; COLEARN_PDL=0 = off): same kernels, same order, so the update must be bit-identical ------------------
_PDL_SCRIPT = """
import hashlib, torch
from colearn_federated_learning_b200.fl.convnet import ConvNetTrainer
from colearn_federated_learning_b200.models.registry import flatten_params
from colearn_federated_learning_b200.models.resnet import ResNet18
dev = torch.device('cuda:0')
torch.manual_seed(0)
x = torch.randn(256, 3, 32, 32, device=dev); y = torch.randint(0, 10, (256,), device=dev)
torch.manual_seed(1)
model = ResNet18(10).to(dev)
flat = flatten_params(model)
tr = ConvNetTrainer(model, dev, 128, (32, 32))
tr.load(flat, model)
for rep in range(3):
    for lo in (0, 128):
        tr._graph_step(x[lo:lo + 128], y[lo:lo + 128], 0.05)
tr.store(flat, model)
torch.cuda.synchronize()
print('HASH', hashlib.sha256(flat.cpu().numpy().tobytes()).hexdigest(), bool(torch.isfinite(flat).all()))
"""


@pytest.mark.parametrize("flags", [{}, {"COLEARN_CONV_WGRAD_MN": "1", "COLEARN_CONV_DGRAD_KN": "1", "COLEARN_CONV_SPLITK": "1",
                                        "COLEARN_CONV_FUSED_BN": "1", "COLEARN_CONV_IMPLICIT": "2"}])
def test_programmatic_dependent_launch_is_bit_identical(flags):
    """Every kernel of the step waits (griddepcontrol.wait) before its first global access, so enabling the attribute may
    only move launch latency, never a value.  The flag is read once per process: two subprocesses."""
    import subprocess
    import sys
    _dev()
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

    def run(pdl):
        env = dict(os.environ, **flags)
        env["COLEARN_PDL"] = "1" if pdl else "0"
        out = subprocess.run([sys.executable, "-c", _PDL_SCRIPT], cwd=root, env=env, capture_output=True, text=True, timeout=300)
        assert out.returncode == 0, out.stderr[-2000:]
        line = [ln for ln in out.stdout.splitlines() if ln.startswith("HASH")][-1].split()
        assert line[2] == "True"
        return line[1]

    assert run(False) == run(True)


# ---- fused wgrad GEMM -> FedAvg reduce (COLEARN_OVERLAP_REDUCE=1 / overlap_reduce=True); tests/test_overlap_reduce.py has the CPU evidence ----
_OVERLAP_SCRIPT = """
import torch
from colearn_federated_learning_b200.data import synthetic_unsw
from colearn_federated_learning_b200.parallel import FederatedEngine
dev = torch.device('cuda:0')
flats, paths = [], []
for overlap in (False, True):
    eng = FederatedEngine('wide_mlp', backend='fused', device=dev, batch_size=128, lr=0.05, seed=6, chunk_elems=4096,
                          bf16_shadow=True, model_kwargs={'width': 512, 'depth': 3}, overlap_reduce=overlap)
    xs, ys = synthetic_unsw(384, seed=20)
    eng.set_local_data(xs, ys)
    rep = eng.run_rounds(3)
    torch.cuda.synchronize()
    flats.append(eng.global_flat().clone())
    paths.append(rep.extra['train_path'])
    assert torch.equal(eng.arena.tensor('shadow')[: eng.P], flats[-1].to(torch.bfloat16))
    if overlap:
        assert bool((eng.prod_count == 0).all())
        assert int(eng.arena.tensor('produced')[: eng.n_chunks].min()) == eng.epoch
assert paths[1].endswith('+overlap_reduce') and not paths[0].endswith('+overlap_reduce'), paths
assert torch.isfinite(flats[1]).all() and torch.equal(flats[0], flats[1])
print('OVERLAP_OK')
"""


@pytest.mark.parametrize("graphs", ["1", "0"])
def test_overlapped_reduce_single_gpu_is_bit_identical(graphs):
    """World 1: the two-shot kernel on the side stream owns every chunk and takes them as the last backward's wgrad
    epilogues (grid capped to leave it its SMs) report them.  Same kernels and order of additions as the serial round.
    (Own process: if a chunk is never reported the kernel's watchdog traps, which kills the CUDA context.)"""
    import subprocess
    import sys
    _dev()
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, COLEARN_CUDA_GRAPHS=graphs, COLEARN_OVERLAP_TIMEOUT_S="5")
    out = subprocess.run([sys.executable, "-c", _OVERLAP_SCRIPT], cwd=root, env=env, capture_output=True, text=True, timeout=240)
    assert out.returncode == 0 and "OVERLAP_OK" in out.stdout, (out.stdout[-1500:], out.stderr[-2500:])


def test_layerwise_trainer_dgrad_against_weights_in_place_on_device():
    """COLEARN_MLP_DGRAD_KN=1: the wide-MLP dgrad reads W_l in place (MN-major B operand) — no W^T copies, no transposes."""
    from colearn_federated_learning_b200.fl import FitConfig
    from colearn_federated_learning_b200.fl.layerwise import LayerwiseMLPTrainer
    from colearn_federated_learning_b200.models import MLPNet, MLPSpec
    dev = _dev()
    torch.manual_seed(0)
    spec = MLPSpec((10, 256, 512, 256, 2), "none", "xent")
    flat0 = flatten_params(MLPNet(spec)).clone().to(dev)
    x, y = torch.rand(384, 10, device=dev), torch.randint(0, 2, (384, 1), device=dev).float()
    cfg = FitConfig(model="x", loss="xent", batch_size=128, lr=0.1)
    outs = []
    for kn in (False, True, "both"):
        flat = flat0.clone()
        tr = LayerwiseMLPTrainer(spec, flat, 128, dgrad_kn=bool(kn), wgrad_mn=(kn == "both"))
        tr.fit(flat, x, y, cfg, None)
        torch.cuda.synchronize()
        outs.append(flat)
    for o in outs[1:]:
        assert torch.isfinite(o).all()
        assert float((outs[0] - o).abs().max()) < 2e-3 * max(1.0, float(outs[0].abs().max()))


def test_star_engine_pipelined_read_back_single_gpu():
    """read_back="pipelined": every round's losses reach the host (one round late), results equal the synchronous mode."""
    from colearn_federated_learning_b200.data import synthetic_unsw
    from colearn_federated_learning_b200.parallel import FederatedEngine
    dev = _dev()
    x, y = synthetic_unsw(300, seed=2)
    hx, hy = x.pin_memory(), y.pin_memory()
    flats, hist = [], None
    for mode in (True, "pipelined"):
        eng = FederatedEngine("mlp", backend="fused", device=dev, batch_size=1, lr=0.05, seed=7, shuffle=False)
        eng.set_local_data(x, y)
        rep = eng.run_rounds(5, host_inputs=[(hx, hy)] * 5, read_back=mode, barrier=False)
        torch.cuda.synchronize()
        flats.append(eng.global_flat().clone())
        if mode == "pipelined":
            hist = torch.stack(eng.loss_history)
            assert hist.shape[0] == 5
            assert torch.allclose(hist[:, :2], rep.losses[:, 0, :].cpu(), atol=0, rtol=0)
            assert torch.equal(eng.loss_host[:2], hist[-1, :2])
    assert torch.equal(flats[0], flats[1])


def test_twoshot_engine_applies_the_server_learning_rate():
    """server_lr != 1 on the large-model (two-shot) path: theta <- theta + lr_s (sum_k w_k theta_k - theta).  The ranks train in
    place on the arena, so the engine keeps the round's starting model; world 1: theta_1 = theta_0 + lr_s (fit(theta_0) - theta_0)."""
    from colearn_federated_learning_b200.data import synthetic_unsw
    from colearn_federated_learning_b200.parallel import FederatedEngine
    dev = _dev()
    xs, ys = synthetic_unsw(256, seed=21)
    outs = {}
    for lr_s in (1.0, 0.5):
        eng = FederatedEngine("wide_mlp", backend="fused", device=dev, batch_size=128, lr=0.05, seed=6, chunk_elems=4096, bf16_shadow=True,
                              model_kwargs={"width": 256, "depth": 3}, server_lr=lr_s)
        eng.set_local_data(xs, ys)
        theta0 = eng.global_flat().clone()
        rep = eng.run_rounds(1)
        torch.cuda.synchronize()
        outs[lr_s] = (theta0, eng.global_flat().clone(), eng.arena.tensor("shadow")[: eng.P].clone())
        assert rep.extra["nvls"] is False
    theta0, full, _ = outs[1.0]
    _, half, shadow = outs[0.5]
    assert torch.equal(outs[0.5][0], theta0) and not torch.equal(full, theta0)
    torch.testing.assert_close(half, theta0 + 0.5 * (full - theta0), rtol=1e-6, atol=1e-7)
    assert torch.equal(shadow, half.to(torch.bfloat16))
