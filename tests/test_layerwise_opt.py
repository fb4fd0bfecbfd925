"""Local optimizers on the layer-wise wgmma trainer (fl/layerwise.py): the optimizer epilogue of gemm_wgmma.cu
(gemm_wgmma_opt_kernel) and local_opt_apply_kernel of elementwise.cu on the SIMT / wgmma host-model build, bit for bit against
reference.local_opt_step on the same GEMM's fp32 product; whole fits of every test_layerwise_general.py case with each optimizer
against torch_fit with the torch.optim optimizer, under that file's bound; fresh state in every fit; plain SGD unchanged; and
the routing.  The GPU twin is test_layerwise_opt_gpu.py."""
import pytest
import torch

import test_layerwise_general as G
import test_local_opt as T
from colearn_federated_learning_b200 import ops
from colearn_federated_learning_b200.fl import FitConfig
from colearn_federated_learning_b200.fl.layerwise import LayerwiseMLPTrainer
from colearn_federated_learning_b200.fl.local_opt import LocalOpt
from colearn_federated_learning_b200.fl.trainer import torch_fit
from colearn_federated_learning_b200.models import MLPNet, MLPSpec, flatten_params, unflatten_params
from colearn_federated_learning_b200.ops import reference as R

simt = T.simt
OPTS = ["momentum", "nesterov_wd", "adam", "adam_wd"]
LR = 0.05
# masters at the edges: zeros of both signs, subnormals, large values
EDGES = [0.0, -0.0, 1e-40, -1e-40, 1.4e-45, 3e30, -3e30, 1e-20]


def _bits_equal(a, b):
    return torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def _opt_arg(lo, state, m, v):
    return [m if (lo.kind == "Adam" or lo.momentum) else None, v if lo.kind == "Adam" else None, lo.launch_args(),
            R.local_opt_scalars(state)]


def _gemm(sim, a, b, mn_m, tile_n, opt=None, **kw):
    args = [a, b, None, False, None, None, kw.get("out_f32"), None, kw.get("sgd_master"), LR, kw.get("sgd_shadow"), None, None,
            tile_n, 0, None, mn_m, False, None, [], []]
    if opt is None:
        sim.gemm_tcgen05(*args)
    else:
        sim.gemm_tcgen05_opt(*args, *opt)


# ---- 1. the optimizer epilogue on the wgmma host model ---------------------------------------------------------------------
@pytest.mark.parametrize("opt", OPTS)
@pytest.mark.parametrize("mn", [False, True])
@pytest.mark.parametrize("tile_n", [128, 256])
def test_epilogue_bits_on_the_host_model(simt, opt, mn, tile_n):
    """Three consecutive steps with carried moments: master, m and v equal the same GEMM's out_f32 followed by the reference
    step, bit for bit; the shadow is the master in bf16"""
    lo = T.OPTS[opt]
    M, N, K = 256, 256, 128
    g = torch.Generator().manual_seed(5 + tile_n + mn)
    master = torch.randn(M, N, generator=g) * 0.3
    master.view(-1)[:len(EDGES)] = torch.tensor(EDGES)
    master.view(-1)[N * 37:N * 37 + len(EDGES)] = torch.tensor(EDGES)
    ref = master.clone()
    m, v = torch.zeros(M, N), torch.zeros(M, N)
    state_k, state_r = R.local_opt_clock(), R.local_opt_state(ref)
    shadow = torch.zeros(M, N, dtype=torch.bfloat16)
    for step in range(3):
        if mn:   # wgrad form: A = dz [K, M], B = a [K, N]
            a, b = torch.randn(K, M, generator=g).to(torch.bfloat16), torch.randn(K, N, generator=g).to(torch.bfloat16)
        else:
            a, b = torch.randn(M, K, generator=g).to(torch.bfloat16), torch.randn(N, K, generator=g).to(torch.bfloat16)
        acc = torch.full((M, N), 7.0)
        _gemm(simt.m, a, b, M if mn else 0, tile_n, out_f32=acc)
        R.local_opt_next(state_k, lo, LR)
        _gemm(simt.m, a, b, M if mn else 0, tile_n, opt=_opt_arg(lo, state_k, m, v), sgd_master=master, sgd_shadow=shadow)
        R.local_opt_step(ref, acc, lo, LR, state_r)
        assert _bits_equal(master, ref), (opt, mn, tile_n, step, (master - ref).abs().max())
        if lo.kind == "Adam" or lo.momentum:
            assert _bits_equal(m, state_r["m"]), (opt, step)
        if lo.kind == "Adam":
            assert _bits_equal(v, state_r["v"]), (opt, step)
        assert torch.equal(shadow, master.to(torch.bfloat16))


def test_epilogue_refusals(simt):
    """The launcher refuses the optimizer epilogue next to every option it does not take, and a missing moment"""
    lo = T.OPTS["adam"]
    st = R.local_opt_clock()
    R.local_opt_next(st, lo, LR)
    a, b = torch.zeros(128, 64, dtype=torch.bfloat16), torch.zeros(128, 64, dtype=torch.bfloat16)
    master, m, v = torch.zeros(128, 128), torch.zeros(128, 128), torch.zeros(128, 128)
    base = [a, b, None, False, None, None, None, None, master, LR, None, None, None, 0, 0, None, 0, False, None, [], []]
    for i, val, what in ((6, torch.zeros(128, 128), "out_"), (12, torch.zeros(4, 128), "colsum"),
                         (14, 2, "split_k"), (2, torch.zeros(128), "bias")):
        args = list(base)
        args[i] = val
        if i == 14:
            args[15] = torch.zeros(2 * 128 * 128)
        with pytest.raises(RuntimeError, match=what):
            simt.m.gemm_tcgen05_opt(*args, m, v, lo.launch_args(), R.local_opt_scalars(st))
    with pytest.raises(RuntimeError, match="keeps it"):
        simt.m.gemm_tcgen05_opt(*base, m, None, lo.launch_args(), R.local_opt_scalars(st))
    with pytest.raises(RuntimeError, match="wgrad"):   # the mn-major dgrad form (b_kn)
        args = list(base)
        args[0], args[1], args[17] = torch.zeros(128, 64, dtype=torch.bfloat16), torch.zeros(64, 128, dtype=torch.bfloat16), True
        simt.m.gemm_tcgen05_opt(*args, m, v, lo.launch_args(), R.local_opt_scalars(st))


# ---- 2. the apply kernel -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("opt", OPTS)
def test_apply_bits_on_strided_blocks(simt, opt):
    """An edge layer [10, 37] inside rows of 48 (the padding columns stay untouched) from a gradient with rows of 128, over
    three steps, bit for bit against the reference step"""
    lo = T.OPTS[opt]
    g = torch.Generator().manual_seed(11)
    rows, cols, ld, g_ld = 10, 37, 48, 128
    store = torch.randn(rows, ld, generator=g)
    store[0, :len(EDGES)] = torch.tensor(EDGES)
    mst, vst = torch.full((rows, ld), 5.0), torch.full((rows, ld), 5.0)
    mst[:, :cols], vst[:, :cols] = 0.0, 0.0
    theta, m, v = store[:, :cols], mst[:, :cols], vst[:, :cols]
    pad = store[:, cols:].clone()
    ref = theta.clone()
    state_k, state_r = R.local_opt_clock(), R.local_opt_state(ref)
    with ops.conv.simt():
        for step in range(3):
            grad = torch.randn(rows, g_ld, generator=g)
            R.local_opt_next(state_k, lo, LR)
            ops.local_opt_apply(theta, grad, (lo, state_k, m if (lo.kind == "Adam" or lo.momentum) else None,
                                              v if lo.kind == "Adam" else None), LR)
            R.local_opt_step(ref, grad[:, :cols].clone(), lo, LR, state_r)
            assert _bits_equal(theta, ref), (opt, step)
            if lo.kind == "Adam" or lo.momentum:
                assert _bits_equal(m, state_r["m"])
            if lo.kind == "Adam":
                assert _bits_equal(v, state_r["v"])
    assert torch.equal(store[:, cols:], pad)
    assert bool((mst[:, cols:] == 5.0).all()) and bool((vst[:, cols:] == 5.0).all())


def _partial_sum(partials, n):
    """bias_sgd_from_partials_kernel's gradient: the partial rows added in order from 0, in float32"""
    g = torch.zeros(n)
    for r in range(partials.shape[0]):
        g = g + partials[r, :n]
    return g


@pytest.mark.parametrize("opt", OPTS)
def test_hidden_bias_from_partials_on_the_simt_build(simt, opt):
    """A hidden bias stepped from the dgrad epilogue's partials [B/32, n_pad]: the gradient is bias_sgd_from_partials's (the
    rows in order; the momentum after the first step is that gradient itself), the step the reference's"""
    lo = T.OPTS[opt]
    g = torch.Generator().manual_seed(3)
    n, n_pad, rows = 130, 256, 12
    bias = torch.randn(n, generator=g)
    ref = bias.clone()
    m, v = torch.zeros(n), torch.zeros(n)
    state_k, state_r = R.local_opt_clock(), R.local_opt_state(ref)
    with ops.conv.simt():
        for step in range(3):
            partials = torch.randn(rows, n_pad, generator=g)
            R.local_opt_next(state_k, lo, LR)
            ops.local_opt_apply(bias.view(1, -1), partials, (lo, state_k, m.view(1, -1), v.view(1, -1) if lo.kind == "Adam" else None),
                                LR, g_rows=rows)
            grad = _partial_sum(partials, n)
            if step == 0 and lo.kind == "SGD" and not lo.weight_decay:
                assert _bits_equal(m, grad)
            R.local_opt_step(ref, grad, lo, LR, state_r)
            assert _bits_equal(bias, ref), (opt, step)


# ---- 3. whole fits against torch.optim ------------------------------------------------------------------------------------
def _torch_opt_case(dims, act, loss, b, n, lo, dev, trainer=None, cfg_kw=None):
    """(trainer's θ, its last loss, torch_fit's θ, its last loss, θ0) for one test_layerwise_general case with optimizer lo"""
    torch.manual_seed(0)
    spec = MLPSpec(tuple(dims), act, loss)
    model = MLPNet(spec)
    flat0 = flatten_params(model).clone()
    x = torch.rand(n, dims[0])
    y = torch.randint(0, dims[-1], (n, 1)).float() if loss == "xent" else (torch.rand(n, dims[-1]) > 0.5).float()
    cfg = FitConfig(model="x", loss=loss, batch_size=b, lr=0.01, epochs=2, **(cfg_kw or {})).with_local_opt(lo)
    perm = R.make_permutation(n, 2, seed=3)
    ref_model = MLPNet(spec)
    unflatten_params(ref_model, flat0.clone())
    ref_last = torch_fit(ref_model, x, y, cfg, perm)
    flat = flat0.clone().to(dev)
    tr = trainer or LayerwiseMLPTrainer(spec, flat, b)
    last = tr.fit(flat, x.to(dev), y.to(dev), cfg, perm.to(dev), local_opt=lo)
    return flat.cpu(), float(last), flatten_params(ref_model), float(ref_last), flat0


def check_against_torch_optim(dims, act, loss, b, n, opt, dev):
    """test_layerwise_general.py's bound (cos > 0.995, rel < 0.1, loss within 5 %), except for Adam: cos > 0.95, rel < 0.35.

    Adam's step is about lr · sign(g) wherever |g| is well above eps, so an entry of the gradient that is a sum of cancelling
    terms gets a full-size step whose sign follows the bf16 rounding of the operands.  `Net` at lr 0.01 measured (CPU definition
    of the trainer against fp32 autograd): Adam cos 0.963 / rel 0.275, Adam with weight decay 0.985 / 0.172, and the BCE case
    with Adam 0.981 / 0.194; all other cases and optimizers stay inside the plain bound.  The rounding alone explains it: the
    same fp32 autograd fit with only x rounded to bf16 moves `Net`'s Adam update by rel 0.216 (momentum: 0.052)."""
    lo = T.FIT_OPTS[opt]
    got, last, ref, ref_last, flat0 = _torch_opt_case(dims, act, loss, b, n, lo, dev)
    upd, upd_ref = got - flat0, ref - flat0
    cos = float((upd * upd_ref).sum() / (upd.norm() * upd_ref.norm()))
    rel = float((upd - upd_ref).norm() / upd_ref.norm())
    cos_min, rel_max = (0.95, 0.35) if lo.kind == "Adam" else (0.995, 0.1)
    assert torch.isfinite(got).all() and cos > cos_min and rel < rel_max, (dims, loss, opt, cos, rel)   # bf16 operands vs fp32
    assert abs(last - ref_last) < 0.05 * max(1.0, abs(ref_last)), (dims, loss, opt, last, ref_last)


@pytest.mark.parametrize("opt", OPTS + ["wd"])
@pytest.mark.parametrize("dims,act,loss,b,n", G.CASES)
def test_fits_match_torch_optim_on_cpu(dims, act, loss, b, n, opt):
    check_against_torch_optim(dims, act, loss, b, n, opt, torch.device("cpu"))


# ---- 4. no state leaks / step counting -------------------------------------------------------------------------------------
def check_fresh_state(dev, opt="adam_wd"):
    """Two consecutive fits on one trainer from the same θ and data give identical bits (moments and step scalars restart)"""
    dims, act, loss, b, n = G.CASES[0]
    spec = MLPSpec(tuple(dims), act, loss)
    torch.manual_seed(0)
    flat0 = flatten_params(MLPNet(spec)).clone().to(dev)
    tr = LayerwiseMLPTrainer(spec, flat0.clone(), b)
    outs = []
    for _ in range(2):
        got, last, _, _, _ = _torch_opt_case(dims, act, loss, b, n, T.FIT_OPTS[opt], dev, trainer=tr)
        outs.append((got, last))
    assert _bits_equal(outs[0][0], outs[1][0]) and outs[0][1] == outs[1][1]


def test_no_state_leaks_between_fits_cpu():
    check_fresh_state(torch.device("cpu"))


@pytest.mark.parametrize("epochs,max_b", [(3, -1), (3, 5), (1, 2), (2, 4)])
def test_step_count_runs_over_the_fit(monkeypatch, epochs, max_b):
    """t runs 1 .. total_steps over the fit's batches across its epochs (ragged tail batches and max_nr_batches included),
    restarting at 1 in the next fit"""
    seen = []
    real = R.local_opt_next

    def spy(state, lo, lr):
        real(state, lo, lr)
        seen.append(state["t"])
    import colearn_federated_learning_b200.fl.layerwise as LW
    monkeypatch.setattr(LW.reference, "local_opt_next", spy)
    dims, act, loss, b, n = G.CASES[1]
    spec = MLPSpec(tuple(dims), act, loss)
    torch.manual_seed(0)
    flat = flatten_params(MLPNet(spec)).clone()
    x, y = torch.rand(n, dims[0]), (torch.rand(n, 1) > 0.5).float()
    cfg = FitConfig(model="x", loss=loss, batch_size=b, lr=0.01, epochs=epochs, max_nr_batches=max_b)
    tr = LayerwiseMLPTrainer(spec, flat, b)
    want = list(range(1, R.total_steps(n, b, epochs, max_b) + 1))
    for _ in range(2):
        seen.clear()
        tr.fit(flat, x, y, cfg, R.make_permutation(n, epochs, seed=1), local_opt=T.OPTS["adam"])
        assert seen == want


# ---- 5. plain SGD unchanged ---------------------------------------------------------------------------------------------
def check_plain_is_unchanged(dev):
    """LocalOpt("SGD", momentum=0, weight_decay=0) and None: the same bits, the same launches, no moments allocated"""
    for dims, act, loss, b, n in G.CASES:
        res = []
        for lo in (None, LocalOpt("SGD", momentum=0.0, weight_decay=0.0)):
            torch.manual_seed(0)
            spec = MLPSpec(tuple(dims), act, loss)
            flat = flatten_params(MLPNet(spec)).clone().to(dev)
            x = torch.rand(n, dims[0])
            y = torch.randint(0, dims[-1], (n, 1)).float() if loss == "xent" else (torch.rand(n, dims[-1]) > 0.5).float()
            tr = LayerwiseMLPTrainer(spec, flat, b)
            last = tr.fit(flat, x.to(dev), y.to(dev), FitConfig(model="x", loss=loss, batch_size=b, lr=0.01, epochs=2),
                          R.make_permutation(n, 2, seed=3).to(dev), local_opt=lo)
            assert tr.opt_m is None and tr.opt_v is None
            res.append((flat.cpu(), float(last), tr.launches))
        assert _bits_equal(res[0][0], res[1][0]) and res[0][1:] == res[1][1:], dims


def test_plain_sgd_is_unchanged_cpu():
    check_plain_is_unchanged(torch.device("cpu"))


def test_momentum_only_keeps_no_v_and_wd_only_keeps_nothing():
    dims, act, loss, b, n = G.CASES[2]
    for opt, has_m, has_v in (("momentum", True, False), ("wd", False, False), ("adam", True, True)):
        spec = MLPSpec(tuple(dims), act, loss)
        flat = flatten_params(MLPNet(spec)).clone()
        tr = LayerwiseMLPTrainer(spec, flat, b)
        tr.fit(flat, torch.rand(n, dims[0]), (torch.rand(n, dims[-1]) > 0.5).float(),
               FitConfig(model="x", loss=loss, batch_size=b, lr=0.01), None, local_opt=T.OPTS[opt])
        assert (tr.opt_m is not None) == has_m and (tr.opt_v is not None) == has_v, opt
        if has_m:
            assert tr.opt_m.numel() == tr.n_params == flat.numel()


# ---- 6. routing ------------------------------------------------------------------------------------------------------------
def test_fused_round_arguments_refuse_an_optimizer():
    """The engine's fused-broadcast / fused-reduce round passes ready / produced / before_last_backward: an optimizer next to
    them is refused before any launch"""
    dims, act, loss, b, n = G.CASES[0]
    spec = MLPSpec(tuple(dims), act, loss)
    flat = flatten_params(MLPNet(spec)).clone()
    tr = LayerwiseMLPTrainer(spec, flat, b)
    cfg = FitConfig(model="x", loss=loss, batch_size=b, lr=0.01)
    for kw in (dict(produced=object()), dict(before_last_backward=lambda: None)):
        with pytest.raises(ValueError, match="plain SGD only"):
            tr.fit(flat, torch.rand(n, dims[0]), torch.zeros(n, 1), cfg, None, local_opt=T.OPTS["momentum"], **kw)


def test_local_fit_passes_the_optimizer_to_the_layerwise_trainer(monkeypatch):
    """local_fit hands a layer-wise MLP's optimizer to the trainer instead of refusing it; the conv-net trainer and the
    two-shot engine path still refuse"""
    from colearn_federated_learning_b200.fl import trainer
    seen = {}

    class Stub:
        launches = 0

        def fit(self, flat, x, y, cfg, perm, local_opt=None):
            seen["lo"] = local_opt
            return torch.zeros(())

    monkeypatch.setattr(LayerwiseMLPTrainer, "cached", staticmethod(lambda *a: Stub()))
    from colearn_federated_learning_b200.models import build_model
    model = build_model("net")
    flat = flatten_params(model)
    # the CUDA branch of local_fit on a CPU box: a flat arena that reports is_cuda
    cuda_flat = torch.Tensor._make_subclass(type("CudaLike", (torch.Tensor,), {"is_cuda": property(lambda self: True)}), flat)
    cfg = FitConfig(model="net", loss="xent", batch_size=32, lr=0.01).with_local_opt(T.OPTS["adam"])
    _, path = trainer.local_fit(cuda_flat, model, torch.rand(64, 1, 28, 28), torch.zeros(64, 1), cfg,
                                perm=R.make_permutation(64, 1, seed=1))
    assert path == "layerwise" and seen["lo"] == T.OPTS["adam"]
    from colearn_federated_learning_b200.parallel.engine import FederatedEngine
    with pytest.raises(ValueError, match="two-shot"):
        FederatedEngine("mlp", backend="cpu", device=torch.device("cpu"), algo="twoshot", local_opt=T.OPTS["adam"])
