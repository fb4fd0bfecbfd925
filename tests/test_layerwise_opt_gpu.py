"""Local optimizers on the layer-wise wgmma trainer, on the H100: the optimizer instances of gemm_wgmma_opt_kernel and
local_opt_apply_kernel bit for bit against the reference step on the same GEMM's fp32 product; whole fits against torch.optim
(test_layerwise_opt.py's bound); fresh state in every fit; plain SGD unchanged; `Net` through local_fit; a few Adam steps of
`wide_mlp`; and the virtual workers of local mode each equal to its shard's fit alone."""
import pytest
import torch

import test_layerwise_general as G
import test_layerwise_opt as LO
import test_local_opt as T
from colearn_federated_learning_b200 import ops
from colearn_federated_learning_b200.fl import FitConfig
from colearn_federated_learning_b200.fl.local_opt import LocalOpt
from colearn_federated_learning_b200.ops import reference as R

gpu = pytest.mark.gpu
DEV = "cuda"


def _moments(lo, m, v):
    return (m if (lo.kind == "Adam" or lo.momentum) else None), (v if lo.kind == "Adam" else None)


@gpu
@pytest.mark.parametrize("opt", LO.OPTS)
@pytest.mark.parametrize("mn", [False, True])
@pytest.mark.parametrize("tile_n", [128, 256])
def test_epilogue_bits_gpu(opt, mn, tile_n):
    """gemm_wgmma_opt_kernel over three steps with carried moments: master, m and v are the same GEMM's out_f32 followed by the
    reference step, bit for bit; the shadow is the master in bf16.  Masters hold 0, -0, subnormal and large values."""
    lo = T.OPTS[opt]
    M, N, K = 512, 512, 256
    g = torch.Generator().manual_seed(7 + tile_n + mn)
    master = torch.randn(M, N, generator=g) * 0.3
    master.view(-1)[:len(LO.EDGES)] = torch.tensor(LO.EDGES)
    ref = master.clone()
    master = master.to(DEV)
    m, v = torch.zeros(M, N, device=DEV), torch.zeros(M, N, device=DEV)
    shadow = torch.zeros(M, N, dtype=torch.bfloat16, device=DEV)
    state_k, state_r = R.local_opt_clock(), R.local_opt_state(ref)
    for step in range(3):
        shape_a, shape_b = ((K, M), (K, N)) if mn else ((M, K), (N, K))
        a = torch.randn(*shape_a, generator=g).to(torch.bfloat16).to(DEV)
        b = torch.randn(*shape_b, generator=g).to(torch.bfloat16).to(DEV)
        acc = torch.full((M, N), 7.0, device=DEV)
        ops.gemm_bf16(a, b, out_f32=acc, tile_n=tile_n, mn_m=M if mn else 0)
        R.local_opt_next(state_k, lo, LO.LR)
        ops.gemm_bf16(a, b, sgd_master=master, sgd_lr=LO.LR, sgd_shadow=shadow, tile_n=tile_n, mn_m=M if mn else 0,
                      opt=(lo, state_k, *_moments(lo, m, v)))
        R.local_opt_step(ref, acc.cpu(), lo, LO.LR, state_r)
        torch.cuda.synchronize()
        assert LO._bits_equal(master.cpu(), ref), (opt, mn, tile_n, step)
        if lo.kind == "Adam" or lo.momentum:
            assert LO._bits_equal(m.cpu(), state_r["m"]), (opt, step)
        if lo.kind == "Adam":
            assert LO._bits_equal(v.cpu(), state_r["v"]), (opt, step)
        assert torch.equal(shadow, master.to(torch.bfloat16))


@gpu
@pytest.mark.parametrize("opt", LO.OPTS)
def test_apply_and_hidden_bias_bits_gpu(opt):
    """local_opt_apply_kernel on a strided edge block (padding untouched) and on a hidden bias from the epilogue partials,
    whose gradient is bias_sgd_from_partials's to the bit"""
    lo = T.OPTS[opt]
    g = torch.Generator().manual_seed(13)
    rows, cols, ld, g_ld = 10, 37, 48, 128
    store = torch.randn(rows, ld, generator=g)
    store[0, :len(LO.EDGES)] = torch.tensor(LO.EDGES)
    ref = store[:, :cols].clone()
    store = store.to(DEV)
    pad = store[:, cols:].clone()
    mst, vst = torch.zeros(rows, ld, device=DEV), torch.zeros(rows, ld, device=DEV)
    state_k, state_r = R.local_opt_clock(), R.local_opt_state(ref)
    for step in range(3):
        grad = torch.randn(rows, g_ld, generator=g)
        R.local_opt_next(state_k, lo, LO.LR)
        ops.local_opt_apply(store[:, :cols], grad.to(DEV), (lo, state_k, *_moments(lo, mst[:, :cols], vst[:, :cols])), LO.LR)
        R.local_opt_step(ref, grad[:, :cols].clone(), lo, LO.LR, state_r)
        assert LO._bits_equal(store[:, :cols].cpu(), ref), (opt, step)
    assert torch.equal(store[:, cols:], pad)
    n, n_pad, prow = 130, 256, 12
    bias = torch.randn(n, generator=g)
    ref = bias.clone()
    bias = bias.to(DEV)
    m, v = torch.zeros(n, device=DEV), torch.zeros(n, device=DEV)
    state_k, state_r = R.local_opt_clock(), R.local_opt_state(ref)
    for step in range(3):
        partials = torch.randn(prow, n_pad, generator=g).to(DEV)
        grad = ops.bias_sgd_from_partials(None, partials, 0.0)[:n].cpu()
        R.local_opt_next(state_k, lo, LO.LR)
        ops.local_opt_apply(bias.view(1, -1), partials, (lo, state_k, *_moments(lo, m.view(1, -1), v.view(1, -1))), LO.LR,
                            g_rows=prow)
        if step == 0 and lo.kind == "SGD" and not lo.weight_decay:
            assert LO._bits_equal(m.cpu(), grad)
        R.local_opt_step(ref, grad, lo, LO.LR, state_r)
        assert LO._bits_equal(bias.cpu(), ref), (opt, step)


@gpu
@pytest.mark.parametrize("opt", LO.OPTS + ["wd"])
@pytest.mark.parametrize("dims,act,loss,b,n", G.CASES)
def test_fits_match_torch_optim_gpu(dims, act, loss, b, n, opt):
    LO.check_against_torch_optim(dims, act, loss, b, n, opt, torch.device(DEV, 0))


@gpu
def test_no_state_leaks_and_plain_sgd_unchanged_gpu():
    LO.check_fresh_state(torch.device(DEV, 0))
    LO.check_fresh_state(torch.device(DEV, 0), "nesterov_wd")
    LO.check_plain_is_unchanged(torch.device(DEV, 0))


@gpu
def test_net_through_local_fit_gpu():
    """`Net` with Adam trains on the layer-wise path; plain SGD named explicitly launches what no optimizer launches, with
    the same bits"""
    from colearn_federated_learning_b200.fl import trainer
    from colearn_federated_learning_b200.models import build_model, flatten_params
    dev = torch.device(DEV, 0)
    torch.manual_seed(0)
    net = build_model("net").to(dev)
    flat0 = flatten_params(net).to(dev)
    x, y = torch.rand(96, 1, 28, 28, device=dev), torch.randint(0, 10, (96, 1), device=dev).float()
    cfg = FitConfig(model="net", loss="xent", batch_size=32, lr=0.01, epochs=2)
    flat = flat0.clone()
    _, path = trainer.local_fit(flat, net, x, y, cfg.with_local_opt(LocalOpt("Adam", eps=1e-3)))
    assert path == "layerwise" and torch.isfinite(flat).all() and not torch.equal(flat, flat0)
    res = []
    for lo in (None, LocalOpt("SGD", momentum=0.0, weight_decay=0.0)):
        f = flat0.clone()
        last, path = trainer.local_fit(f, net, x, y, cfg.with_local_opt(lo))
        res.append((f.cpu(), float(last), trainer.LAST_FIT_LAUNCHES, path))
    assert torch.equal(res[0][0], res[1][0]) and res[0][1:] == res[1][1:]


@gpu
def test_wide_mlp_adam_steps_gpu():
    """Four batch-128 Adam steps of `wide_mlp` (BASELINE config 5; the exact 4096-wide layers take the wgmma optimizer
    epilogue): finite, the same bits in two runs, and within the Adam bound of torch_fit on the same GPU"""
    from colearn_federated_learning_b200.fl.trainer import local_fit, torch_fit
    from colearn_federated_learning_b200.models import build_model, flatten_params, unflatten_params
    dev = torch.device(DEV, 0)
    torch.manual_seed(0)
    model = build_model("wide_mlp").to(dev)
    flat0 = flatten_params(model).to(dev).clone()
    n = 512
    x, y = torch.rand(n, 10, device=dev), torch.randint(0, 2, (n, 1), device=dev).float()
    lo = LocalOpt("Adam", eps=1e-3)
    cfg = FitConfig(model="wide_mlp", loss="xent", batch_size=128, lr=1e-3, epochs=1).with_local_opt(lo)
    perm = ops.device_permutation(n, 1, seed=4, device=dev)
    outs = []
    for _ in range(2):
        flat = flat0.clone()
        last, path = local_fit(flat, model, x, y, cfg, perm=perm)
        assert path == "layerwise"
        outs.append((flat, float(last)))
    assert torch.isfinite(outs[0][0]).all() and torch.equal(outs[0][0], outs[1][0]) and outs[0][1] == outs[1][1]
    ref_model = build_model("wide_mlp").to(dev)
    unflatten_params(ref_model, flat0.clone())
    ref_last = float(torch_fit(ref_model, x, y, cfg, perm))
    upd, upd_ref = (outs[0][0] - flat0).double(), (flatten_params(ref_model) - flat0).double()
    cos = float((upd * upd_ref).sum() / (upd.norm() * upd_ref.norm()))
    rel = float((upd - upd_ref).norm() / upd_ref.norm())
    assert cos > 0.95 and rel < 0.35, (cos, rel)
    assert abs(outs[0][1] - ref_last) < 0.05 * max(1.0, abs(ref_last)), (outs[0][1], ref_last)


@gpu
def test_virtual_workers_are_their_shards_fits_gpu():
    """train_virtual_workers with `Net` on CUDA and Adam: every worker's model is its shard's local_fit alone, bit for bit"""
    from types import SimpleNamespace
    from colearn_federated_learning_b200.control.coordinator import train_virtual_workers
    from colearn_federated_learning_b200.fl.trainer import local_fit
    from colearn_federated_learning_b200.models import build_model, flatten_params
    dev = torch.device(DEV, 0)
    torch.manual_seed(0)
    model = build_model("net").to(dev)
    theta = flatten_params(model).to(dev).clone()
    g = torch.Generator().manual_seed(2)
    shards = {f"w{i}": SimpleNamespace(x=torch.rand(k, 1, 28, 28, generator=g).to(dev),
                                        y=torch.randint(0, 10, (k, 1), generator=g).float().to(dev)) for i, k in enumerate((70, 0, 45))}

    class _Shard:
        def __init__(self, s):
            self.x, self.y = s.x, s.y

        def __len__(self):
            return self.x.shape[0]

    class Fed:
        workers = list(shards)

        def __getitem__(self, k):
            return _Shard(shards[k])
    cfg = FitConfig(model="net", loss="xent", batch_size=32, epochs=2, lr=0.01, seed=5).with_local_opt(LocalOpt("Adam", eps=1e-3))
    flats, losses, counts = train_virtual_workers(theta.clone(), model, Fed(), cfg, 0)
    assert counts == [70, 0, 45]
    assert torch.equal(flats[1], theta)
    for i, wid in enumerate(Fed.workers):
        if counts[i] == 0:
            continue
        alone = theta.clone()
        last, path = local_fit(alone, model, shards[wid].x, shards[wid].y, cfg.with_seed(cfg.seed + 31 * i), 0)
        assert path == "layerwise"
        assert torch.equal(flats[i], alone) and losses[i] == float(last), wid
