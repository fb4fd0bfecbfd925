"""Fused wgrad GEMM → FedAvg reduce (ops/produced.py, csrc/produced.cuh): host-side bookkeeping on the PyTorch definitions,
then the whole round — layer-wise trainer, epilogue reports, overlapped two-shot — from the kernel SOURCES on the CPU
(SIMT shim + functional wgmma model).  The GPU run of the same path is in tests/test_gpu_schedules.py."""
import pytest
import torch

from colearn_federated_learning_b200.fl import FitConfig
from colearn_federated_learning_b200.fl.layerwise import LayerwiseMLPTrainer
from colearn_federated_learning_b200.models import MLPNet, MLPSpec
from colearn_federated_learning_b200.models.registry import flatten_params
from colearn_federated_learning_b200.ops.produced import ProducedSpec


def _arena(spec, seed, extra=12):
    torch.manual_seed(seed)
    flat = flatten_params(MLPNet(spec)).clone()
    n = (flat.numel() + 3) // 4 * 4 + extra                     # + a tail the parameters do not cover
    arena = torch.zeros(n)
    arena[: flat.numel()] = flat
    return arena, flat.numel()


@pytest.mark.parametrize("chunk", [256, 4096, 65536])
def test_last_backward_reports_every_arena_element_exactly_once(chunk):
    spec = MLPSpec((10, 128, 256, 2), "none", "xent")            # edge layers (padded) + one exact layer
    cfg = FitConfig(model="x", loss="xent", batch_size=128, lr=0.1)
    arena, P = _arena(spec, 0)
    base = arena.clone()
    torch.manual_seed(1)
    x, y = torch.rand(384, 10), torch.randint(0, 2, (384, 1)).float()
    n = arena.numel()
    n_chunks = (n + chunk - 1) // chunk
    W, rank = 3, 1
    tables = torch.zeros(W, W, n_chunks, dtype=torch.int32)
    epoch = torch.tensor([4], dtype=torch.int32)
    sp = ProducedSpec.reference(tables, epoch, 1, chunk_elems=chunk, n=n, rank=rank)
    calls = []
    tr = LayerwiseMLPTrainer(spec, arena[:P], 128)

    def before_last():
        # nothing has been reported when the overlapped two-shot is launched
        calls.append(int(tables.abs().sum()))

    tr.fit(arena[:P], x, y, cfg, None, produced=sp, before_last_backward=before_last)
    assert calls == [0]
    assert sp.idle()
    for c in range(n_chunks):
        assert int(tables[c % W, rank, c]) == 5
    assert int((tables != 0).sum()) == n_chunks                  # nothing outside the owners' rows of this producer
    # same parameters as a fit without the reports
    tr2 = LayerwiseMLPTrainer(spec, base[:P], 128)
    tr2.fit(base[:P], x, y, cfg, None)
    assert torch.equal(arena, base)


def test_reference_spec_rejects_double_reports():
    tables = torch.zeros(2, 2, 4, dtype=torch.int32)
    sp = ProducedSpec.reference(tables, torch.tensor([0], dtype=torch.int32), 1, chunk_elems=64, n=256, rank=0)
    sp.mark(0, 100)
    with pytest.raises(AssertionError):
        sp.mark(60, 120)


def test_round_from_kernel_sources_with_overlapped_reduce():
    """Two emulated ranks, wide-MLP round: the last backward's wgrad GEMMs (kernel source on the wgmma model) report
    their blocks, the overlapped two-shot kernel (kernel source on the SIMT shim) reduces on the produced tables alone;
    result = FedAvg of two independent plain fits."""
    from colearn_federated_learning_b200.ops import conv as conv_ops
    simt = conv_ops.load_simt()
    if simt is None or not hasattr(simt, "produced_mark"):
        pytest.skip("SIMT build unavailable")
    spec = MLPSpec((10, 128, 128, 2), "none", "xent")
    cfg = FitConfig(model="x", loss="xent", batch_size=128, lr=0.1)
    W, chunk = 2, 2048
    arenas, data = [], []
    for r in range(W):
        a, P = _arena(spec, 0, extra=0)                            # same initial model on both ranks
        arenas.append(a)
        torch.manual_seed(10 + r)
        data.append((torch.rand(256, 10), torch.randint(0, 2, (256, 1)).float()))
    n = arenas[0].numel()
    n_chunks = (n + chunk - 1) // chunk
    works = torch.stack(arenas).contiguous()
    plain = works.clone()
    tables = torch.zeros(W, W, n_chunks, dtype=torch.int32)
    epoch = torch.tensor([0], dtype=torch.int32)
    with conv_ops.simt():
        for r in range(W):
            count = torch.zeros(n_chunks, dtype=torch.int32)
            sp = ProducedSpec.device(simt, count, [tables[o].data_ptr() for o in range(W)], epoch, 1, chunk_elems=chunk, n=n, rank=r,
                                     max_ctas=2)
            tr = LayerwiseMLPTrainer(spec, works[r, :P], 128)
            tr.fit(works[r, :P], data[r][0], data[r][1], cfg, None, produced=sp)
            assert sp.idle()
            tr2 = LayerwiseMLPTrainer(spec, plain[r, :P], 128)
            tr2.fit(plain[r, :P], data[r][0], data[r][1], cfg, None)
    torch.testing.assert_close(works, plain, rtol=0, atol=0)
    assert int(tables.min(dim=1).values.sum()) >= 0 and all(int(tables[c % W, k, c]) == 1 for c in range(n_chunks) for k in range(W))
    weights = torch.tensor([0.5, 0.5])
    flags = torch.zeros(W, n_chunks, dtype=torch.int32)
    arrive = torch.zeros(W, dtype=torch.int32)
    for r in range(W):
        simt.twoshot_fedavg(r, works, None, flags, arrive, weights, None, 1, 0b11, 1.0, chunk, 2, tables, 10.0)
    want = plain.mean(0)
    for k in range(W):
        torch.testing.assert_close(works[k], want, rtol=1e-6, atol=1e-6)


# ---- layer-wise trainer without W^T copies (COLEARN_MLP_DGRAD_KN=1): dgrad reads W_l in place as an MN-major B operand -------------
def test_layerwise_dgrad_against_weights_in_place():
    from colearn_federated_learning_b200.ops import conv as conv_ops
    spec = MLPSpec((10, 128, 256, 128, 2), "none", "xent")
    cfg = FitConfig(model="x", loss="xent", batch_size=128, lr=0.1)
    torch.manual_seed(5)
    x, y = torch.rand(256, 10), torch.randint(0, 2, (256, 1)).float()
    a0, P = _arena(spec, 3, extra=0)
    a1, a2 = a0.clone(), a0.clone()
    LayerwiseMLPTrainer(spec, a0[:P], 128, dgrad_kn=False).fit(a0[:P], x, y, cfg, None)
    tr = LayerwiseMLPTrainer(spec, a1[:P], 128, dgrad_kn=True)
    assert all(t is None for t in tr.WsT)                       # no transposed copies exist
    tr.fit(a1[:P], x, y, cfg, None)
    assert torch.equal(a0, a1)                                   # definitions: same products, same order
    simt = conv_ops.load_simt()
    if simt is None or not hasattr(simt, "gemm_tcgen05"):
        pytest.skip("SIMT build unavailable")
    with conv_ops.simt():                                        # kernel source: MN-major B operand on the wgmma model
        LayerwiseMLPTrainer(spec, a2[:P], 128, dgrad_kn=True).fit(a2[:P], x, y, cfg, None)
    torch.testing.assert_close(a2, a0, rtol=2e-3, atol=2e-3)


def test_layerwise_wgrad_from_untransposed_operands():
    """COLEARN_MLP_WGRAD_MN=1 (+ DGRAD_KN): no transposed activation / gradient / weight copy exists any more."""
    from colearn_federated_learning_b200.ops import conv as conv_ops
    spec = MLPSpec((10, 128, 256, 128, 2), "none", "xent")
    cfg = FitConfig(model="x", loss="xent", batch_size=128, lr=0.1)
    torch.manual_seed(6)
    x, y = torch.rand(256, 10), torch.randint(0, 2, (256, 1)).float()
    a0, P = _arena(spec, 4, extra=0)
    a1, a2 = a0.clone(), a0.clone()
    LayerwiseMLPTrainer(spec, a0[:P], 128, dgrad_kn=False, wgrad_mn=False).fit(a0[:P], x, y, cfg, None)
    tr = LayerwiseMLPTrainer(spec, a1[:P], 128, dgrad_kn=True, wgrad_mn=True)
    assert all(t is None for t in tr.WsT + tr.aT + tr.dzT)
    tr.fit(a1[:P], x, y, cfg, None)
    assert torch.equal(a0, a1)
    simt = conv_ops.load_simt()
    if simt is None or not hasattr(simt, "gemm_tcgen05"):
        pytest.skip("SIMT build unavailable")
    with conv_ops.simt():                                        # kernel source: MN-major A and B operands + fused SGD epilogue
        LayerwiseMLPTrainer(spec, a2[:P], 128, dgrad_kn=True, wgrad_mn=True).fit(a2[:P], x, y, cfg, None)
    torch.testing.assert_close(a2, a0, rtol=2e-3, atol=2e-3)


def test_transposes_are_refreshed_on_demand_and_never_after_the_last_step(monkeypatch):
    """W^T is only rebuilt when a dgrad needs it: a fit of S steps launches (S - 1) x L weight transposes behind its
    wgrads instead of S x L (the ones after the last step were dead work: the next fit starts from refresh_exact)."""
    from colearn_federated_learning_b200.fl import layerwise as lw_mod
    spec = MLPSpec((10, 128, 256, 128, 2), "none", "xent")
    cfg = FitConfig(model="x", loss="xent", batch_size=128, lr=0.1)
    torch.manual_seed(7)
    x, y = torch.rand(384, 10), torch.randint(0, 2, (384, 1)).float()
    a0, P = _arena(spec, 5, extra=0)
    tr = LayerwiseMLPTrainer(spec, a0[:P], 128, dgrad_kn=False, wgrad_mn=False)      # the K-major form: W^T copies exist
    calls = []
    real = lw_mod.ops.transpose_bf16

    def counting(src, out=None):
        calls.append(src.data_ptr())
        return real(src, out)

    monkeypatch.setattr(lw_mod.ops, "transpose_bf16", counting)
    tr.fit(a0[:P], x, y, cfg, None)                              # 3 steps
    L = spec.n_layers
    w_ptrs = {w.data_ptr() for w in tr.Ws}
    n_w = sum(1 for c in calls if c in w_ptrs)
    # fit start: L refreshes; then dgrads of steps 2 and 3 refresh layers 1 .. L-1 (layer 0 has no dgrad)
    assert n_w == L + 2 * (L - 1), (n_w, calls)
    assert not any(tr._wt_fresh[1:])                             # stale after the last wgrad ...
    tr.sync_transposes()                                         # ... until somebody asks
    for l in range(L):
        assert torch.equal(tr.WsT[l], tr.Ws[l].t().contiguous())
    # two consecutive fits == one trainer doing the same steps with eager transposes (reference: recompute from scratch)
    b0, _ = _arena(spec, 5, extra=0)
    tr2 = LayerwiseMLPTrainer(spec, b0[:P], 128, dgrad_kn=False, wgrad_mn=False)
    tr2.fit(b0[:P], x, y, cfg, None)
    assert torch.equal(a0, b0)
    tr.fit(a0[:P], x, y, cfg, None)
    tr2.sync_transposes()
    tr2.fit(b0[:P], x, y, cfg, None)
    assert torch.equal(a0, b0)
