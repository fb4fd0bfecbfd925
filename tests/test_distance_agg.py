"""Distance-based robust aggregation (the weighted geometric median ``geomed`` and the norm-bounded mean ``norm_clip``,
``ops/csrc/distance_agg.cuh``) without a GPU: the PyTorch definition against an independent float64 transcription, its
semantics, the kernel sources on the SIMT CPU build against the definition, and the argument / Coordinator plumbing.

Tolerances.  The distances are float64 sums of float32 differences: the definition and the kernels form them bit for bit
alike, and they differ from a float64 Weiszfeld only through the float32 centre (one rounding per fmaf, K fmaf per element:
relative error <= K 2^-24 of the centre's magnitude).  The weights then agree to ~1e-6 relative, and the aggregate to a few
float32 ulps of the rows' magnitude: ``atol = rtol = 2e-5`` with rows of magnitude ~1 and K <= 100.  The reference adds
with separate multiply and add roundings where the kernels use fmaf, hence the same tolerance between the SIMT build and the
reference; two launch grids of the SIMT build give identical bits."""
import math

import numpy as np
import pytest
import torch

from colearn_federated_learning_b200 import ops
from colearn_federated_learning_b200.fl.aggregate import Aggregator
from colearn_federated_learning_b200.fl.server_opt import ServerOpt
from colearn_federated_learning_b200.fl.uplink import UplinkCodec
from colearn_federated_learning_b200.ops import reference

TOL = dict(atol=2e-5, rtol=2e-5)
GEO = Aggregator("geomed", iters=3)
CLIP = Aggregator("norm_clip", clip_norm=2.0)


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


def rows_around(K, P, seed, spread=0.1):
    g = torch.Generator().manual_seed(seed)
    theta = torch.randn(P, generator=g)
    return theta, theta + spread * torch.randn(K, P, generator=g)


def np_weiszfeld(x, alpha, c0, iters, eps):
    """float64 smoothed Weiszfeld from c0, the excluded rows as in the definition"""
    x, alpha, c = x.astype(np.float64), alpha.astype(np.float64), c0.astype(np.float64)
    for _ in range(iters):
        d = np.sqrt(((x - c) ** 2).sum(1))
        b = np.where(np.isfinite(d), alpha / np.maximum(eps, np.where(np.isfinite(d), d, 1.0)), 0.0)
        c = (b[:, None] * np.where(np.isfinite(x), x, 0.0)).sum(0) / b.sum()
    return c


def np_clipped(x, alpha, c0, tau):
    x, alpha, c0 = x.astype(np.float64), alpha.astype(np.float64), c0.astype(np.float64)
    d = np.sqrt(((x - c0) ** 2).sum(1))
    ok = np.isfinite(d)
    a = np.where(ok, alpha, 0.0) / np.where(ok, alpha, 0.0).sum()
    b = a * np.minimum(1.0, tau / np.where(ok & (d > 0), d, 1.0))
    return c0 + (b[:, None] * np.where(ok[:, None], x - c0, 0.0)).sum(0)


# ---- the definition ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("K,P", [(1, 100), (5, 2401), (16, 5000), (40, 4097)])
def test_reference_matches_float64(K, P):
    theta, x = rows_around(K, P, K + P)
    alpha = torch.rand(K, generator=torch.Generator().manual_seed(1)) + 0.1
    alpha /= alpha.sum()
    a, _ = reference.distance_aggregate(x, alpha, Aggregator("geomed", iters=4, eps=1e-6), theta)
    np.testing.assert_allclose(a.numpy(), np_weiszfeld(x.numpy(), alpha.numpy(), theta.numpy(), 4, 1e-6), **TOL)
    a, _ = reference.distance_aggregate(x, alpha, Aggregator("norm_clip", clip_norm=0.5), theta)
    np.testing.assert_allclose(a.numpy(), np_clipped(x.numpy(), alpha.numpy(), theta.numpy(), 0.5), **TOL)


def test_distances_are_float64_sums_of_float32_differences():
    theta, x = rows_around(3, 9000, 2)
    d2 = reference.distance_sq(x, theta)
    exact = ((x - theta).double() ** 2).sum(1)
    assert torch.allclose(d2, exact, rtol=1e-13, atol=0)


def test_semantics():
    theta, x = rows_around(6, 3000, 3)
    u = torch.full((6,), 1 / 6)
    for agg in (GEO, CLIP):
        a, w = reference.distance_aggregate(x[:1], torch.ones(1), agg, theta)                   # K = 1: the row (norm_clip: clipped)
        if agg is GEO:
            assert torch.equal(a, x[0]) and float(w[0]) == 1.0
        same = x[:1].repeat(4, 1)
        a, _ = reference.distance_aggregate(same, torch.full((4,), 0.25), GEO, theta)          # identical rows: that row
        assert torch.allclose(a, x[0], atol=1e-6)
        bad = torch.cat([x, torch.full((1, 3000), float("nan")), torch.full((1, 3000), float("inf"))])
        bad[7, 5] = float("inf")
        ab, wb = reference.distance_aggregate(bad, torch.full((8,), 1 / 8), agg, theta)
        af, wf = reference.distance_aggregate(x, u, agg, theta)
        assert torch.allclose(ab, af, atol=1e-6) and float(wb[6]) == 0.0 and float(wb[7]) == 0.0
        assert torch.isfinite(ab).all()
        allbad = torch.full((3, 3000), float("nan"))
        a0, w0 = reference.distance_aggregate(allbad, torch.full((3,), 1 / 3), agg, theta)     # nothing left: the start point
        assert torch.equal(a0, theta) and not w0.any()
    # norm_clip with every update inside tau is the weighted mean
    a, _ = reference.distance_aggregate(x, u, Aggregator("norm_clip", clip_norm=1e6), theta)
    assert torch.allclose(a, reference.fedavg_flat(x, u), atol=1e-5)
    # a x1000 update moves the aggregate by at most alpha_k tau beyond the others
    boosted = x.clone()
    boosted[2] = theta + 1000 * (x[2] - theta)
    tau = 2.0
    a_b, w_b = reference.distance_aggregate(boosted, u, Aggregator("norm_clip", clip_norm=tau), theta)
    others = theta + sum(w_b[k] * (boosted[k] - theta) for k in range(6) if k != 2)
    assert float((a_b - others).norm()) <= u[2] * tau * (1 + 1e-3)
    assert float(w_b[2]) < 1e-3 * float(w_b[0])
    # --weighted changes geomed
    aw, _ = reference.distance_aggregate(x, torch.tensor([0.5, 0.3, 0.05, 0.05, 0.05, 0.05]), GEO, theta)
    au, _ = reference.distance_aggregate(x, u, GEO, theta)
    assert not torch.allclose(aw, au, atol=1e-4)


def test_geomed_is_robust_to_far_rows():
    g = torch.Generator().manual_seed(4)
    mu = torch.randn(2000, generator=g)
    honest = mu + 0.1 * torch.randn(10, 2000, generator=g)
    far = mu + 50.0 + torch.randn(4, 2000, generator=g)
    x = torch.cat([honest, far])
    u = torch.full((14,), 1 / 14)
    mean_err = float((reference.fedavg_flat(x, u) - mu).norm())
    geo_err = float((reference.distance_aggregate(x, u, Aggregator("geomed", iters=8), mu)[0] - mu).norm())
    # honest spread: 0.1 sqrt(2000) ~ 4.5 per row; the mean is dragged ~ 4/14 * 50 sqrt(2000) ~ 640 away
    assert mean_err > 500 and geo_err < 10, (mean_err, geo_err)


# ---- the kernels on the SIMT CPU build ---------------------------------------------------------------------------------------
def _simt_apply(simt, theta, x, alpha, agg, opt=None, grid=0, codec=None, payload=None, scales=None):
    w_out = torch.zeros(x.shape[0] if x is not None else payload.shape[0])
    if opt is None:
        okind, hyper, m, v, lr = 0, [], None, None, 1.0
    else:
        okind, hyper, m, v, lr = opt.code, opt.hyper, opt.m, opt.v, opt.lr
    tail = dict(agg_kind=agg.code, trim=0.0, iters=agg.iters, eps=agg.eps, clip=agg.clip, agg_weights_out=w_out, grid=grid)
    if codec is None:
        simt.fedavg_apply(theta, x, alpha, lr, okind, hyper, m, v, **tail)
    else:
        simt.fedavg_apply_quantized(theta, payload, scales, alpha, codec.bits, lr, okind, hyper, m, v, **tail)
    return w_out


CASES = [(1, 1001), (2, 2048), (5, 2401), (8, 1001), (16, 3 * 4096), (32, 2401), (33, 2048), (100, 1001)]


@pytest.mark.parametrize("K,P", CASES)
@pytest.mark.parametrize("agg", [GEO, CLIP], ids=["geomed", "norm_clip"])
def test_simt_fp32_matches_reference(simt, K, P, agg):
    theta, x = rows_around(K, P, 10 * K + P)
    if K > 2:
        x[1] = float("nan")
        x[2] *= 1000
    alpha = torch.rand(K, generator=torch.Generator().manual_seed(K)) + 0.5
    alpha /= alpha.sum()
    want = theta.clone()
    w_ref = torch.zeros(K)
    ops.fedavg_apply(want, x, alpha, aggregator=agg, agg_weights_out=w_ref)
    got = theta.clone()
    w = _simt_apply(simt, got, x, alpha, agg)
    torch.testing.assert_close(got, want, **TOL)
    torch.testing.assert_close(w, w_ref, atol=1e-6, rtol=1e-5)
    assert torch.isfinite(got).all()


@pytest.mark.parametrize("bits", [8, 4])
@pytest.mark.parametrize("K,P", [(1, 1001), (5, 2401), (16, 2048), (33, 3 * 4096), (100, 1001)])
@pytest.mark.parametrize("agg", [GEO, CLIP], ids=["geomed", "norm_clip"])
def test_simt_quantized_matches_reference(simt, K, P, bits, agg):
    theta, x = rows_around(K, P, K * P + bits)
    codec = UplinkCodec(f"int{bits}")
    payload, scales = reference.encode_delta(x, theta, bits, list(range(1, K + 1)))
    if K > 2:
        scales[1, 0] = float("nan")                    # a non-finite block: the row is excluded
    alpha = torch.full((K,), 1.0 / K)
    want = theta.clone()
    w_ref = torch.zeros(K)
    ops.fedavg_apply_quantized(want, payload, scales, alpha, codec, aggregator=agg, agg_weights_out=w_ref)
    got = theta.clone()
    w = _simt_apply(simt, got, None, alpha, agg, codec=codec, payload=ops._aligned_rows(payload), scales=scales.contiguous())
    torch.testing.assert_close(got, want, **TOL)
    torch.testing.assert_close(w, w_ref, atol=1e-6, rtol=1e-5)
    if K > 2:
        assert float(w[1]) == 0.0


@pytest.mark.parametrize("kind", ["sgd", "adam"])
@pytest.mark.parametrize("agg", [GEO, CLIP], ids=["geomed", "norm_clip"])
def test_simt_misaligned_theta_with_server_opt(simt, kind, agg):
    K, P = 7, 2401
    base, x = rows_around(K, P + 1, 5)
    theta_buf = base.clone()
    theta = theta_buf[1:]                                 # 4-byte offset: the scalar paths
    x = x[:, 1:].contiguous()
    alpha = torch.full((K,), 1.0 / K)
    opt = ServerOpt(kind, lr=0.5 if kind == "sgd" else 0.01)
    st_ref, st = opt.init_state(P, "cpu"), opt.init_state(P, "cpu")
    want = theta.clone()
    ops.fedavg_apply(want, x, alpha, opt=st_ref, aggregator=agg)
    got = theta
    _simt_apply(simt, got, x, alpha, agg, opt=st)
    torch.testing.assert_close(got, want, **TOL)
    torch.testing.assert_close(st.m, st_ref.m, **TOL)


@pytest.mark.parametrize("agg", [GEO, Aggregator("geomed", iters=5), CLIP], ids=["geomed3", "geomed5", "norm_clip"])
def test_simt_grid_independent(simt, agg):
    K, P = 6, 3 * 4096 + 5
    theta, x = rows_around(K, P, 6)
    alpha = torch.full((K,), 1.0 / K)
    outs = []
    for grid in (1, 3, 0):
        t = theta.clone()
        w = _simt_apply(simt, t, x, alpha, agg, grid=grid)
        outs.append((t, w))
    for t, w in outs[1:]:
        assert torch.equal(t.view(torch.int32), outs[0][0].view(torch.int32))
        assert torch.equal(w.view(torch.int32), outs[0][1].view(torch.int32))


def test_simt_distances_bit_exact(simt):
    """one geomed step (L = 1) is c^1 = sum fmaf(w_k, x_k): its weights come from the distances to theta, which the definition
    forms bit for bit"""
    K, P = 9, 5000
    theta, x = rows_around(K, P, 9)
    alpha = torch.full((K,), 1.0 / K)
    _, w_ref = reference.distance_aggregate(x, alpha, Aggregator("geomed", iters=1), theta)
    w = _simt_apply(simt, theta.clone(), x, alpha, Aggregator("geomed", iters=1))
    assert torch.equal(w.view(torch.int32), w_ref.view(torch.int32))


# ---- arguments, refusals, Coordinator ----------------------------------------------------------------------------------------
def _cli(*argv):
    import federated_coordinator as fc
    return fc.arguments_from_cli(fc.parse_cli(["-t", "topic/state", *argv]))


def test_aggregator_validation():
    assert Aggregator("geomed").iters == 3 and Aggregator("geomed").eps == 1e-6
    for bad in (dict(kind="norm_clip"), dict(kind="norm_clip", clip_norm=0.0), dict(kind="norm_clip", clip_norm=math.inf),
                dict(kind="geomed", iters=0), dict(kind="geomed", iters=17), dict(kind="geomed", eps=0.0),
                dict(kind="geomed", eps=float("nan")), dict(kind="geomed", eps=1e-50)):
        with pytest.raises(ValueError):
            Aggregator(**bad)
    a = Aggregator("geomed")
    assert a.robust and a.distance_based and a.weighted and not a.coordinate_wise
    assert Aggregator("median").coordinate_wise and not Aggregator("median").weighted


def test_cli_flags_and_refusals():
    agg = _cli("--aggregator", "geomed", "--geomed-iters", "5", "--geomed-eps", "1e-4", "--weighted").client_aggregator()
    assert (agg.kind, agg.iters, agg.eps) == ("geomed", 5, 1e-4)
    agg = _cli("--aggregator", "norm_clip", "--clip-norm", "3", "--weighted").client_aggregator()
    assert (agg.kind, agg.clip) == ("norm_clip", 3.0)
    for bad in (["--aggregator", "norm_clip"], ["--aggregator", "geomed", "--geomed-iters", "0"],
                ["--aggregator", "geomed", "--geomed-eps", "-1"], ["--aggregator", "geomed", "--uplink-codec", "topk"],
                ["--aggregator", "geomed", "--box"], ["--aggregator", "norm_clip", "--clip-norm", "1", "-r", "--secure-agg"]):
        with pytest.raises(SystemExit):
            _cli(*bad)


def test_refusal_messages_name_the_reason():
    from colearn_federated_learning_b200.control.arguments import Arguments
    a = Arguments(aggregator="geomed", uplink="topk")
    with pytest.raises(ValueError, match="sparse deltas would measure"):
        a.uplink_codec()
    a = Arguments(aggregator="geomed", secure_agg=True)
    with pytest.raises(ValueError, match="distances it weighs by"):
        a.secagg_clip_value()
    codec = UplinkCodec("topk", k=8)
    with pytest.raises(ValueError, match="which entries the codec kept"):
        ops.fedavg_apply_topk(torch.zeros(10), torch.zeros(1, 8, dtype=torch.uint8), torch.zeros(1, 8), torch.ones(1), codec, aggregator=GEO)
    with pytest.raises(ValueError, match="masks hide"):
        ops.fedavg_apply_secagg(torch.zeros(10), torch.zeros(1, 10, dtype=torch.int32), [], [], 8, 1, aggregator=CLIP)
    from colearn_federated_learning_b200.parallel.engine import FederatedEngine
    with pytest.raises(ValueError, match="not available in the multi-GPU engine"):
        FederatedEngine.__init__(object.__new__(FederatedEngine), aggregator=GEO)
    with pytest.raises(ValueError, match="unweighted"):                      # the coordinate-wise refusal is unchanged
        Arguments(aggregator="median", weighted=True).client_aggregator()


def _local_run(tmp_path, argv, patch=None, monkeypatch=None):
    from colearn_federated_learning_b200.control import coordinator as coord_mod
    from colearn_federated_learning_b200.control.bus import BusClient, InProcessBroker
    from colearn_federated_learning_b200.control.window import FakeClock
    from colearn_federated_learning_b200.models import FFNN, flatten_params
    from colearn_federated_learning_b200.utils.checkpoint import save_model

    if patch is not None:
        orig = coord_mod.train_virtual_workers

        def patched(*a, **kw):
            flats, losses, counts = orig(*a, **kw)
            flats = flats.clone()
            patch(flats)
            return flats, losses, counts
        monkeypatch.setattr(coord_mod, "train_virtual_workers", patched)
    args = _cli(*argv, "--synthetic", "90", "--lr", "0.05")
    broker, clock = InProcessBroker(), FakeClock()
    c = coord_mod.Coordinator(1, False, 2, False, False, args=args, broker=broker, timer_factory=clock, path=str(tmp_path / "m.pth"),
                              device=torch.device("cpu"))
    c.connect()
    c.subscribe("topic/state")
    pub = BusClient("pub", broker=broker)
    pub.connect()
    torch.manual_seed(0)
    save_model(FFNN(), c.path)
    for ip in ["10.0.0.1", "10.0.0.2", "10.0.0.3"]:
        pub.publish("topic/state", f"({ip}, TRAINING)")
    c.drain()
    clock.advance(1.0)
    m = FFNN()
    m.load_state_dict(torch.load(c.path, weights_only=True))
    return flatten_params(m), c.metrics.records


@pytest.mark.parametrize("argv", [["--aggregator", "geomed", "--weighted"], ["--aggregator", "norm_clip", "--clip-norm", "0.5"]])
@pytest.mark.parametrize("bad", ["nan", "boost"])
def test_local_mode_with_a_bad_worker(tmp_path, monkeypatch, argv, bad):
    clean, recs = _local_run(tmp_path / "a", argv)
    assert len(recs) == 2 and all(len(r["agg_weights"]) == 3 for r in recs)

    def spoil(flats):
        if bad == "nan":
            flats[1] = float("nan")
        else:
            flats[1] = flats[1] * 1000
    theta, recs = _local_run(tmp_path / "b", argv, spoil, monkeypatch)
    assert torch.isfinite(theta).all()
    if bad == "nan":
        assert all(r["agg_weights"][1] == 0.0 for r in recs)
    # the aggregate stays near the run whose worker behaved; far from what the mean would have done
    assert float((theta - clean).norm()) < 0.5 * float(clean.norm()), float((theta - clean).norm())


def test_distance_kernels_do_not_spill():
    """ptxas -v of the build: no spill in any instance of the distance-based passes (every centre path, fp32 / int8 / int4)"""
    import os
    import re
    path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "colearn_federated_learning_b200", "ops", "csrc",
                        "_obj", "elementwise.cu.log")
    if not os.path.exists(path):
        pytest.skip("needs the build's ptxas log (run the build first)")
    lines = open(path).read().splitlines()
    found = {}
    for i, line in enumerate(lines):
        m = re.search(r"Compiling entry function '(\S+)' for 'sm_90a'", line)
        if m and "dagg_" in m.group(1):
            spill = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", " ".join(lines[i + 1: i + 4]))
            found[m.group(1)] = int(spill.group(1)) + int(spill.group(2))
    centre = [k for k in found if "dagg_center_kernel" in k]
    assert len(centre) == 12, sorted(found)              # KMAX 0 / 4 / 8 / 16 x fp32 / int8 / int4
    assert len([k for k in found if "dagg_apply_kernel" in k]) == 12 and len([k for k in found if "dagg_dist_kernel" in k]) == 3
    assert all(v == 0 for v in found.values()), found


def test_remote_mode_geomed_int8_weighted(tmp_path):
    """remote mode over TCP workers (the harness of tests/test_uplink_quant.py) with --aggregator geomed --uplink-codec int8
    --weighted: the rounds complete and record every device's final weight"""
    from colearn_federated_learning_b200.control.arguments import Arguments
    from test_uplink_quant import _make, _worker
    args = Arguments(model="mlp", lr=0.1, batch_size=16, federate_after_n_batches=30, uplink="int8", synthetic=64, aggregator="geomed",
                     weighted=True)
    torch.manual_seed(0)
    workers = [_worker(1), _worker(2)]
    try:
        c, pub, clock = _make(tmp_path, args, 2)
        for _, port in workers:
            pub.publish("topic/state", f"(127.0.0.1, {port}, TRAINING)")
        c.drain()
        clock.advance(1.0)
        res = c.windower.last_result
    finally:
        for w, _ in workers:
            w.stop()
    assert res is not None and res["dropped"] == [] and all(w.fits_served == 2 for w, _ in workers)
    recs = [r for r in c.metrics.records if "agg_weights" in r]
    assert len(recs) == 2
    for r in recs:
        assert len(r["agg_weights"]) == 2 and all(w > 0 for w in r["agg_weights"]) and abs(sum(r["agg_weights"]) - 1) < 1e-5
