"""The layer-wise wgmma trainer covers every MLP shape the persistent kernel does not: hidden widths and batch sizes
that are not multiples of 128 (zero padding / zero-gradient rows), a short last batch, and the BCE / SSE / MSE heads —
compared with plain autograd on the same sample order.  CPU run = the PyTorch definitions of the ops (same orchestration);
the GPU case runs the kernels."""
import pytest
import torch

from colearn_federated_learning_b200.fl import FitConfig
from colearn_federated_learning_b200.fl.layerwise import LayerwiseMLPTrainer
from colearn_federated_learning_b200.fl.trainer import local_fit, torch_fit
from colearn_federated_learning_b200.models import MLPNet, MLPSpec, flatten_params, unflatten_params
from colearn_federated_learning_b200.ops import reference as R

CASES = [((784, 128, 64, 10), "none", "xent", 32, 100),        # the reference's `Net` (cf.py:22-34): 64-wide layer, batch 32, ragged tail
         ((10, 200, 96, 1), "sigmoid", "bce", 50, 120),        # BCE head, nothing a multiple of 128, short last batch (20 rows)
         ((12, 130, 3), "none", "sse", 128, 256),              # SSE on a linear head
         ((12, 130, 3), "sigmoid", "mse", 16, 40)]


def _case(dims, act, loss, b, n, dev):
    torch.manual_seed(0)
    spec = MLPSpec(tuple(dims), act, loss)
    model = MLPNet(spec)
    flat0 = flatten_params(model).clone()
    x = torch.rand(n, dims[0])
    y = torch.randint(0, dims[-1], (n, 1)).float() if loss == "xent" else (torch.rand(n, dims[-1]) > 0.5).float()
    cfg = FitConfig(model="x", loss=loss, batch_size=b, lr=0.01, epochs=2)   # (bf16 noise of a 4-row tail batch grows with lr)
    perm = R.make_permutation(n, 2, seed=3)
    assert LayerwiseMLPTrainer.supports(spec, cfg)
    ref_model = MLPNet(spec)
    unflatten_params(ref_model, flat0.clone())
    ref_last = torch_fit(ref_model, x, y, cfg, perm)
    ref = flatten_params(ref_model)
    flat = flat0.clone().to(dev)
    tr = LayerwiseMLPTrainer(spec, flat, b)
    assert tr.B % 128 == 0 and tr.b == b and tr.n_steps(n, cfg) == 2 * -(-n // b)
    last = tr.fit(flat, x.to(dev), y.to(dev), cfg, perm.to(dev))
    upd, upd_ref = flat.cpu() - flat0, ref - flat0
    cos = float((upd * upd_ref).sum() / (upd.norm() * upd_ref.norm()))
    rel = float((upd - upd_ref).norm() / upd_ref.norm())
    assert torch.isfinite(flat).all() and cos > 0.995 and rel < 0.1, (cos, rel)       # bf16 operands vs fp32 autograd
    assert abs(float(last) - float(ref_last)) < 0.05 * max(1.0, abs(float(ref_last)))


@pytest.mark.parametrize("dims,act,loss,b,n", CASES)
def test_general_mlp_shapes_match_autograd_on_cpu(dims, act, loss, b, n):
    _case(dims, act, loss, b, n, torch.device("cpu"))


@pytest.mark.gpu
@pytest.mark.parametrize("dims,act,loss,b,n", CASES)
def test_general_mlp_shapes_match_autograd_on_gpu(dims, act, loss, b, n):
    _case(dims, act, loss, b, n, torch.device("cuda", 0))


@pytest.mark.gpu
def test_cuda_tensors_never_fall_back_to_autograd_silently(monkeypatch):
    """`Net` on a GPU trains on the wgmma layer-wise path; a ResNet shard the conv kernels do not cover raises instead of
    switching to cuDNN, unless the library path is requested explicitly."""
    from colearn_federated_learning_b200.models import build_model
    dev = torch.device("cuda", 0)
    monkeypatch.delenv("COLEARN_ALLOW_AUTOGRAD", raising=False)
    monkeypatch.delenv("COLEARN_CONV_PATH", raising=False)
    net = build_model("net").to(dev)
    flat = flatten_params(net).to(dev)
    x, y = torch.rand(96, 1, 28, 28, device=dev), torch.randint(0, 10, (96, 1), device=dev).float()
    _, path = local_fit(flat, net, x, y, FitConfig(model="net", loss="xent", batch_size=32, lr=0.05))
    assert path == "layerwise"
    res = build_model("resnet18").to(dev)
    rflat = flatten_params(res).to(dev)
    xi, yi = torch.randn(100, 3, 32, 32, device=dev), torch.randint(0, 10, (100, 1), device=dev).float()
    with pytest.raises(RuntimeError, match="no sm_90a kernel path"):
        local_fit(rflat, res, xi, yi, FitConfig(model="resnet18", loss="xent", batch_size=100, lr=0.05))
    monkeypatch.setenv("COLEARN_CONV_PATH", "torch")
    _, path = local_fit(rflat, res, xi, yi, FitConfig(model="resnet18", loss="xent", batch_size=100, lr=0.05))
    assert path == "torch"
