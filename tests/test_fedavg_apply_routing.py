"""The one fused FedAvg launcher (``launch_fedavg_apply``) over its whole routing grid, through the SIMT CPU build:
{fp32, int8, int4, topk, secagg} rows x {mean, median, trimmed_mean, geomed, norm_clip} x {sgd, adam}, with K = 3 (register
paths) and K = 40 (the general robust path and the general geomed centre pass).

An admitted cell must match ``ops`` on CPU tensors (``ops.reference``) within the tolerance of that format's own test
(bit-exact for secure aggregation).  A refused cell (top-k or secure-aggregation rows with anything but the mean) must raise
the ``ops`` ValueError, and the binding called with the same arguments must fail in the launcher without touching theta."""
import numpy as np
import pytest
import torch

from colearn_federated_learning_b200 import ops
from colearn_federated_learning_b200.fl.aggregate import Aggregator
from colearn_federated_learning_b200.fl.server_opt import ServerOpt
from colearn_federated_learning_b200.fl.uplink import UplinkCodec
from colearn_federated_learning_b200.ops import reference

P = 1001                                   # partial last 256-block and 2048-chunk
AGGS = {"mean": Aggregator("mean"), "median": Aggregator("median"), "trimmed_mean": Aggregator("trimmed_mean", 0.2),
        "geomed": Aggregator("geomed", iters=3), "norm_clip": Aggregator("norm_clip", clip_norm=2.0)}
REFUSED = {("topk", "median"): "only the \\(weighted\\) mean does", ("topk", "trimmed_mean"): "only the \\(weighted\\) mean does",
           ("topk", "geomed"): "which entries the codec kept", ("topk", "norm_clip"): "which entries the codec kept",
           ("secagg", "median"): "only learns the sum", ("secagg", "trimmed_mean"): "only learns the sum",
           ("secagg", "geomed"): "distances it weighs by", ("secagg", "norm_clip"): "distances it weighs by"}


@pytest.fixture(scope="module")
def simt():
    import importlib.util
    import os
    import shutil

    from colearn_federated_learning_b200.ops import build
    if shutil.which("g++") is None or not os.path.exists(os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include", "cuda_runtime.h")):
        pytest.skip("no g++ / CUDA headers on this box: the SIMT emulator cannot be built")
    path = build.build_simt_emul()
    spec = importlib.util.spec_from_file_location("_colearn_simt", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _padded(payload):
    """the payload with 16-byte rows, as the kernels take it"""
    out = torch.zeros(payload.shape[0], (payload.shape[1] + 15) // 16 * 16, dtype=torch.uint8)
    out[:, :payload.shape[1]] = payload
    return out


def _cell(fmt, K):
    """(ops apply bound to its rows, the SIMT binding, its leading arguments after theta), and theta"""
    g = torch.Generator().manual_seed(K * 7 + len(fmt))
    theta = torch.randn(P, generator=g)
    models = theta + 0.1 * torch.randn(K, P, generator=g)
    models[1] *= 30                                                  # one far row for the robust kinds to act on
    w = torch.rand(K, generator=g) + 0.5
    w /= w.sum()
    if fmt == "fp32":
        return (lambda t, **kw: ops.fedavg_apply(t, models, w, **kw)), "fedavg_apply", [models, w], theta
    if fmt in ("int8", "int4"):
        codec = UplinkCodec(fmt)
        payload, scales = ops.encode_delta(models, theta, codec, list(range(K)))
        return ((lambda t, **kw: ops.fedavg_apply_quantized(t, payload, scales, w, codec, **kw)), "fedavg_apply_quantized",
                [_padded(payload), scales, w, codec.bits], theta)
    if fmt == "topk":
        codec = UplinkCodec("topk", k=8)
        idx, val = ops.encode_topk_delta(models, theta, torch.zeros(K, P), codec)
        return (lambda t, **kw: ops.fedavg_apply_topk(t, idx, val, w, codec, **kw)), "fedavg_apply_topk", [idx, val, w, codec.k], theta
    rng = np.random.default_rng(K)
    keys = [bytes(rng.integers(0, 256, 32, dtype=np.uint8)) for _ in range(K + 2)]
    signs = [1 if i % 3 else -1 for i in range(K + 2)]
    masked = torch.randint(-2 ** 31, 2 ** 31, (K, P), generator=g, dtype=torch.int64).to(torch.int32)
    kw_, sg = ops.secagg_key_words(keys), torch.tensor(signs, dtype=torch.int32)
    return ((lambda t, **kw: ops.fedavg_apply_secagg(t, masked, keys, signs, 23, K + 1, **kw)), "fedavg_apply_secagg",
            [masked, kw_, sg, 23, K + 1], theta)


def _same(a, b):
    return torch.equal(a.view(torch.int32), b.view(torch.int32))


@pytest.mark.parametrize("K", [3, 40])
@pytest.mark.parametrize("opt_kind", ["sgd", "adam"])
@pytest.mark.parametrize("agg_name", list(AGGS))
@pytest.mark.parametrize("fmt", ["fp32", "int8", "int4", "topk", "secagg"])
def test_every_cell_of_the_routing_grid(simt, fmt, agg_name, opt_kind, K):
    agg = AGGS[agg_name]
    apply, binding, lead, theta = _cell(fmt, K)
    opt = ServerOpt("adam", lr=0.05) if opt_kind == "adam" else None
    st_ref, st = (opt.init_state(P), opt.init_state(P)) if opt else (None, None)
    step = dict(opt=st_ref) if opt else dict(server_lr=0.7)
    w_ref, w_got = torch.zeros(K), torch.zeros(K)
    tail = ([float(opt.lr), opt.code, opt.hyper, st.m, st.v] if opt else [0.7, 0, [], None, None])
    tail += [agg.code, agg.trim, agg.iters, agg.eps, agg.clip, w_got if agg.distance_based else None, 0]
    got = theta.clone()
    if (fmt, agg_name) in REFUSED:
        with pytest.raises(ValueError, match=REFUSED[fmt, agg_name]):
            apply(theta.clone(), aggregator=agg, **step)
        with pytest.raises(RuntimeError, match="launch failed"):
            getattr(simt, binding)(got, *lead, *tail)
        assert torch.equal(got, theta)
        return
    extra = dict(agg_weights_out=w_ref) if agg.distance_based else {}
    want = apply(theta.clone(), aggregator=agg, **step, **extra)
    getattr(simt, binding)(got, *lead, *tail)
    if fmt == "secagg":
        assert _same(got, want) and (opt is None or (_same(st.m, st_ref.m) and _same(st.v, st_ref.v)))
        return
    tol = dict(atol=2e-5, rtol=2e-5) if agg.distance_based else dict(atol=1e-5, rtol=1e-5)
    torch.testing.assert_close(got, want, **tol)
    if opt:
        torch.testing.assert_close(st.m, st_ref.m, **tol)
        torch.testing.assert_close(st.v, st_ref.v, rtol=1e-5, atol=1e-7)
    if agg.distance_based:
        torch.testing.assert_close(w_got, w_ref, atol=1e-6, rtol=1e-5)
