"""The kernels of csrc/elementwise.cu that every round and every evaluation goes through, at the edges where kernels go
wrong: past the persistent grid (a second grid-stride pass), off 16-byte alignment (the scalar paths), K > 256 FedAvg
weights, tails of 1-3 elements, and the special values (NaN, +-inf, +-0, subnormals, bf16 ties).

Two kinds of reference:
* exact, for the kernels with a fixed operation order (sgd_step, scale_inplace, fedavg_flat / fedavg_apply,
  bias_sgd_from_partials, fp32_to_bf16, transpose_bf16, feistel_permutation, minmax_scale): the GPU bits must equal a
  correctly rounded evaluation of the same operations.  ``fmaf_exact`` is that evaluation of fmaf for numpy arrays; the
  CPU group checks it against libm's fmaf in the SIMT build of the same kernel source.
* float64 with an error model, for the losses and eval, whose __expf / __logf are approximations on the GPU only:
  ``expf_rel`` / ``logf_abs`` / ``sum_rel`` below hold the bounds, and every such test reports its largest error as a
  fraction of its bound (printed at the end of the module: run with ``-s`` to see it).

The CPU group (no mark) runs the special-value cases through the kernel sources compiled for the CPU (host_shim.h).
"""
import math

import numpy as np
import pytest
import torch

from colearn_federated_learning_b200 import ops
from colearn_federated_learning_b200.models import FFNN, MLP, flatten_params
from colearn_federated_learning_b200.ops import reference as R

F32, F64 = np.float32, np.float64
U = 2.0 ** -24                        # unit roundoff of fp32
ULP1 = 2.0 ** -23                     # one ulp relative to a value's leading bit (ulp(x) <= 2^-23 |x|)
GRID_CAP = 132 * 8                    # grid_for's CTA cap
THREADS = 256
VEC_WRAP = GRID_CAP * THREADS * 4     # 1,081,344: first element of the vector kernels' second grid-stride pass
SCALAR_WRAP = GRID_CAP * THREADS      # 270,336: loss / eval / permutation kernels (one element per thread)
ROW_WRAP = GRID_CAP * THREADS // 32   # 8,448 rows: one warp per row
N_SIZES = [1, 3, 4, 5, VEC_WRAP - 1, VEC_WRAP + 5, 4 * 2 ** 20 + 3]
NAN, INF = float("nan"), float("inf")

gpu = pytest.mark.gpu
FRACTIONS = {}     # kernel -> largest |error| / bound seen


def _record(name, frac):
    FRACTIONS[name] = max(FRACTIONS.get(name, 0.0), float(frac))


@pytest.fixture(scope="module", autouse=True)
def _report_fractions():
    yield
    if FRACTIONS:
        print("\nlargest error / error-model bound: " + ", ".join(f"{k} {v:.3g}" for k, v in sorted(FRACTIONS.items())))


def _build_simt():
    import importlib.util
    import os
    import shutil

    from colearn_federated_learning_b200.ops import build
    if shutil.which("g++") is None or not os.path.exists(os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include", "cuda_runtime.h")):
        return None
    path = build.build_simt_emul()
    spec = importlib.util.spec_from_file_location("_colearn_simt", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.fixture(scope="module")
def simt():
    mod = _build_simt()
    if mod is None:
        pytest.skip("no g++ / CUDA headers on this box: the SIMT emulator cannot be built")
    return mod


def _dev():
    return torch.device("cuda", 0)


# ---- exact references ----------------------------------------------------------------------------------------------
def fmaf_exact(a, b, c) -> np.ndarray:
    """fmaf(a, b, c) correctly rounded, elementwise over fp32 arrays.  a * b is exact in float64 (24 + 24 bits); the sum
    is taken to float64 with round-to-odd (TwoSum gives its exact error, and an inexact even result moves to its odd
    neighbour towards the error), and a round-to-odd result with 53 >= 24 + 2 bits rounds to fp32 as the exact value
    would.  (Plain float64 then fp32 rounds twice and is 1 ulp off in rare halfway cases.)"""
    a, b, c = np.broadcast_arrays(*(np.asarray(v, F32).astype(F64) for v in (a, b, c)))
    p = a * b
    s = p + c
    bv = s - p
    err = (p - (s - bv)) + (c - bv)
    s = np.array(s, copy=True)
    fix = (err != 0) & ((s.view(np.uint64) & 1) == 0)
    s[fix] = np.nextafter(s[fix], np.where(err[fix] > 0, np.inf, -np.inf))
    return s.astype(F32)


def _ordered(x):
    i = np.asarray(x, F32).view(np.int32).astype(np.int64)
    return np.where(i < 0, -(i & 0x7FFFFFFF), i)


def ulps(a, b):
    """distance in fp32 ulps (+0 and -0 are 0 apart)"""
    return np.abs(_ordered(a) - _ordered(b))


def assert_bits(got, want, what=""):
    got, want = np.asarray(got, F32), np.asarray(want, F32)
    assert got.shape == want.shape, what
    same = (got.view(np.uint32) == want.view(np.uint32)) | (np.isnan(got) & np.isnan(want))
    if not same.all():
        i = int(np.flatnonzero(~same.reshape(-1))[0])
        raise AssertionError(f"{what}: {int((~same).sum())} of {same.size} differ, first at {i}: {got.reshape(-1)[i]!r} vs {want.reshape(-1)[i]!r}")


def _np(t):
    return t.detach().cpu().numpy()


# ---- the error model of the GPU's intrinsics -----------------------------------------------------------------------
def expf_rel(x):
    """relative error bound of __expf(x): 2 + floor(1.173 |x|) ulp (CUDA math API), one ulp <= 2^-23 of the value"""
    x = np.abs(np.asarray(x, F64))
    return np.where(np.isfinite(x), (2 + np.floor(1.173 * np.where(np.isfinite(x), x, 0))) * ULP1, 0.0)


def logf_abs(x):
    """absolute error bound of __logf(x): 2^-21.41 on [0.5, 2], 3 ulp of the result elsewhere"""
    x = np.asarray(x, F64)
    with np.errstate(divide="ignore", invalid="ignore"):
        lg = np.abs(np.log(x))
    return np.where((x >= 0.5) & (x <= 2.0), 2.0 ** -21.41, 3 * ULP1 * np.where(np.isfinite(lg), lg, 0))


def log1pf_abs(v):
    """log1pf is an IEEE-accurate function on the GPU (1 ulp); bound it by 2 ulp of the result"""
    v = np.abs(np.asarray(v, F64))
    return 2 * ULP1 * np.where(np.isfinite(v), v, 0)


def sum_rel(terms_per_thread, tree_levels, serial_atomics):
    """relative error bound (x sum of |terms|) of an fp32 reduction: a thread's sequential adds, the shuffle / shared tree,
    then the atomicAdds of the blocks (or warps) into one float, in any order: a chain of that many roundings"""
    return (terms_per_thread + tree_levels + serial_atomics + 2) * U


def _grid(n, per_thread=1):
    return max(1, min(GRID_CAP, -(-n // (THREADS * per_thread))))


def _bce_floor(x):
    return np.where(x < -100.0, -100.0, x)          # keeps NaN, -inf -> -100


# ====================================================================================================================
# CPU group: the special-value cases through the kernel sources (SIMT build)
# ====================================================================================================================
def _argmax_special_rows(cols):
    rows = []
    base = np.linspace(-1, 1, cols).astype(F32)
    rows.append(np.full(cols, 2.5, F32))                                  # all tied -> 0
    r = base.copy(); r[cols // 2] = NAN; rows.append(r)                    # one NaN
    rows.append(np.full(cols, NAN, F32))                                  # all NaN -> 0
    rows.append(np.full(cols, -INF, F32))                                 # all -inf -> 0
    r = base.copy(); r[-1] = INF; rows.append(r)                          # +inf
    r = np.zeros(cols, F32); r[0] = -0.0; rows.append(r)                  # -0.0 == +0.0 -> 0
    r = np.full(cols, -0.0, F32); r[-1] = 0.0; rows.append(r)
    if cols > 8:
        r = base.copy(); r[[cols - 1, 7]] = NAN; rows.append(r)            # NaNs in two lanes: the lower index wins
        r = base.copy(); r[[3, cols - 2]] = NAN; r[cols - 1] = INF; rows.append(r)
    if cols > 33:
        r = base.copy(); r[[33, 1]] = NAN; rows.append(r)                 # one lane's two NaNs
        r = base.copy(); r[[40, 8]] = 7.0; rows.append(r)                 # a tie across lanes 8 / 8 (same lane) and more
        r = base.copy(); r[[35, 2]] = 7.0; rows.append(r)                 # a tie across lanes 3 / 2
    r = base.copy(); r[0] = NAN; rows.append(r)
    r = base.copy(); r[-1] = NAN; rows.append(r)
    return np.stack(rows)


@pytest.mark.parametrize("cols", [1, 2, 31, 32, 33, 70])
def test_argmax_special_values_kernel_source(simt, cols):
    x = torch.from_numpy(_argmax_special_rows(cols))
    assert torch.equal(simt.argmax_rows(x.contiguous()), x.argmax(1, keepdim=True))


def test_bce_keeps_nan_kernel_source(simt):
    z = torch.tensor([0.0, 1e-8, -1e-8, 15, -15, 20, -20, 88, -88, 89, -89, 1e4, -1e4, INF, -INF])
    for t in (0.0, 1.0):
        y = torch.full_like(z, t)
        loss, dz = simt.sigmoid_bce(z, y)
        want, wdz = R.sigmoid_bce(z, y)
        assert math.isfinite(float(loss))                                  # +-inf and +-1e4 still clamp to -100
        assert abs(float(loss) - float(want)) <= 1e-5 * abs(float(want)) + 1e-6
        torch.testing.assert_close(dz, wdz, rtol=0, atol=1e-7)
        zn = torch.cat([z, torch.tensor([NAN])])
        loss, dz = simt.sigmoid_bce(zn, torch.full_like(zn, t))
        assert math.isnan(float(loss)) and math.isnan(float(R.sigmoid_bce(zn, torch.full_like(zn, t))[0]))
        assert torch.isnan(dz[-1]) and torch.isfinite(dz[:-1]).all()
    p = torch.tensor([0.0, 1.0, 0.5, 1 - 2 ** -24, 2 ** -126, 0.25])
    y = torch.tensor([1.0, 0.0, 1.0, 1.0, 1.0, 0.0])
    loss, correct = simt.eval_binary(p, y)
    want, wc = R.eval_binary(p, y)
    assert abs(float(loss) - float(want)) <= 1e-6 * abs(float(want)) and int(correct) == int(wc) == 2
    loss, correct = simt.eval_binary(torch.cat([p, torch.tensor([NAN])]), torch.cat([y, torch.tensor([1.0])]))
    assert math.isnan(float(loss)) and int(correct) == 2


def test_minmax_special_values_kernel_source(simt):
    x = torch.tensor([[1.0, 5.0, NAN, 3.0, NAN],
                      [NAN, 5.0, NAN, -1.0, 2.0],
                      [3.0, 5.0, NAN, 1e30, -2.0],
                      [2.0, 5.0, NAN, -1e30, 0.0]])
    got = simt.minmax_scale(x)
    cpu = ops.minmax_scale(x)
    assert torch.equal(torch.isnan(got), torch.isnan(x)) and torch.equal(torch.isnan(cpu), torch.isnan(x))
    fin = ~torch.isnan(x)
    assert (ulps(_np(got[fin]), _np(cpu[fin])) <= 1).all()
    assert got[0, 0] == 0 and got[2, 0] == 1 and (got[:, 1] == 0).all()   # NaN left out of min / max; constant column -> 0
    assert got[3, 3] == 0 and got[2, 3] == 1 and got[1, 4] == 1 and got[2, 4] == 0


def test_fmaf_reference_against_libm(simt):
    """fmaf_exact == libm fmaf (sgd_step's fmaf(-lr, g, p) in the SIMT build), also on sums built to be halfway cases"""
    g = np.random.default_rng(0)
    n = 200_003
    p = g.standard_normal(n).astype(F32)
    gr = g.standard_normal(n).astype(F32)
    # halfway-prone: p + g with g a few ulps of p off a power of two, and products with long tails
    p[:1000] = F32(1.0)
    gr[:1000] = (g.integers(1, 1 << 12, 1000) * 2.0 ** -36).astype(F32)
    lr = 0.3
    pt = torch.from_numpy(p.copy())
    simt.sgd_step(pt, torch.from_numpy(gr), lr)
    assert_bits(_np(pt), fmaf_exact(-F32(lr), gr, p), "libm fmaf vs fmaf_exact")
    double_rounded = (p.astype(F64) - F64(F32(lr)) * gr.astype(F64)).astype(F32)
    assert (ulps(double_rounded, _np(pt)) <= 1).all()


# ====================================================================================================================
# GPU group
# ====================================================================================================================
@pytest.fixture(scope="module")
def simt_or_none():
    return _build_simt()


def _views(n, offset, fill=NAN, dtype=torch.float32, rng=None):
    """a length-n view at element `offset` of a larger buffer (offsets 1-3 break 16-byte alignment); the rest holds `fill`"""
    buf = torch.full((n + 8,), fill, dtype=dtype, device=_dev())
    return buf, buf[offset:offset + n]


@gpu
@pytest.mark.parametrize("n", N_SIZES)
def test_sgd_step_bits(n, simt_or_none):
    g = np.random.default_rng(n)
    p0 = g.standard_normal(n).astype(F32)
    gr = (g.standard_normal(n) * np.exp(g.uniform(-20, 5, n))).astype(F32)
    lr = 0.0123
    want = fmaf_exact(-F32(lr), gr, p0)
    assert (ulps(want, p0.astype(F64) - F64(F32(lr)) * gr.astype(F64)) <= 1).all()          # checks the reference itself
    if simt_or_none is not None and n <= VEC_WRAP + 5:
        pt = torch.from_numpy(p0.copy())
        simt_or_none.sgd_step(pt, torch.from_numpy(gr), lr)
        assert_bits(_np(pt), want, "SIMT sgd_step")
    for po, go in ((0, 0), (1, 0), (0, 2), (3, 3), (2, 1)):
        pbuf, p = _views(n, po)
        gbuf, gv = _views(n, go)
        p.copy_(torch.from_numpy(p0))
        gv.copy_(torch.from_numpy(gr))
        ops.sgd_step(p, gv, lr)
        torch.cuda.synchronize()
        assert_bits(_np(p), want, f"sgd_step p+{po} g+{go}")
        assert torch.isnan(pbuf[:po]).all() and torch.isnan(pbuf[po + n:]).all()       # nothing outside the view
    # bf16 gradient (its own scalar kernel)
    gb = torch.from_numpy(gr).to(torch.bfloat16)
    for po in (0, 1):
        pbuf, p = _views(n, po)
        p.copy_(torch.from_numpy(p0))
        ops.sgd_step(p, gb.to(_dev()), lr)
        torch.cuda.synchronize()
        assert_bits(_np(p), fmaf_exact(-F32(lr), _np(gb.float()), p0), f"sgd_step bf16 grad p+{po}")


@gpu
@pytest.mark.parametrize("n", N_SIZES)
def test_scale_inplace_bits(n):
    g = np.random.default_rng(n + 1)
    p0 = (g.standard_normal(n) * np.exp(g.uniform(-30, 30, n))).astype(F32)
    p0[: min(n, 4)] = np.array([0.0, -0.0, 1e-45, -3e-39], F32)[: min(n, 4)]          # zeros and subnormals
    for scale in (0.3, 0.0, 1.0):
        want = p0 * F32(scale)                                                         # one correctly rounded product
        assert (ulps(want, p0.astype(F64) * F64(F32(scale))) <= 1).all()
        for off in (0, 1, 3):
            buf, p = _views(n, off)
            p.copy_(torch.from_numpy(p0))
            ops._ext.require().scale_inplace(p.data_ptr(), n, scale)
            torch.cuda.synchronize()
            assert_bits(_np(p), want, f"scale_inplace x{scale} +{off}")
            assert torch.isnan(buf[:off]).all() and torch.isnan(buf[off + n:]).all()


def _fedavg_chain(slots, w, theta=None, server_lr=1.0):
    acc = np.zeros(slots.shape[1], F32)
    for c in range(slots.shape[0]):
        acc = fmaf_exact(w[c], slots[c], acc)
    if theta is None:
        return acc
    return fmaf_exact(F32(server_lr), acc - theta, theta)


@gpu
@pytest.mark.parametrize("k,n", [(1, 4099), (2, 4099), (7, 4099), (256, 4099), (257, 4099), (300, 4099), (300, 4096),
                                 (3, 1), (3, 3), (3, 4), (3, 5), (2, VEC_WRAP - 1), (3, VEC_WRAP + 5), (2, 4 * 2 ** 20 + 3),
                                 (257, 300_001)])
def test_fedavg_bits_on_every_path(k, n, simt_or_none):
    """fedavg_flat and fedavg_apply: the fmaf chain in slot order from +0 then theta += lr (a - theta), bit for bit on the
    vector path (16-byte aligned, stride % 4 == 0, scalar tail), the stride path (slots wider than theta, stride % 4 in
    1..3) and the misaligned-theta path; weights past the 256 staged in shared memory, a zero weight, sum != 1"""
    g = np.random.default_rng(k * 7 + n)
    slots = g.standard_normal((k, n)).astype(F32)
    w = (g.uniform(0.1, 1.0, k) / k * 1.3).astype(F32)
    if k > 1:
        w[k // 2] = 0.0
    if k > 256:
        w[256:] *= 5                          # make the weights beyond the staged ones count
    theta0 = g.standard_normal(n).astype(F32)
    flat = _fedavg_chain(slots, w)
    bound = (k + 1) * U * (np.abs(w[:, None].astype(F64) * slots).sum(0))
    assert (np.abs(flat - (w[:, None].astype(F64) * slots).sum(0)) <= bound).all()           # the reference vs float64
    dev = _dev()
    wt = torch.from_numpy(w).to(dev)
    st = torch.from_numpy(slots).to(dev)
    assert_bits(_np(ops.fedavg_flat(st, wt)), flat, "fedavg_flat")
    if simt_or_none is not None and k * n <= 2_000_000:
        assert_bits(_np(simt_or_none.fedavg_flat(torch.from_numpy(slots), torch.from_numpy(w))), flat, "SIMT fedavg_flat")
    w4 = -(-n // 4) * 4
    for server_lr in (1.0, 0.7):
        want = _fedavg_chain(slots, w, theta0, server_lr)
        if simt_or_none is not None and k * n <= 2_000_000:
            th = torch.from_numpy(theta0.copy())
            simt_or_none.fedavg_apply(th, torch.from_numpy(slots), torch.from_numpy(w), server_lr)
            assert_bits(_np(th), want, "SIMT fedavg_apply")
        # (width, theta offset): vector path, three stride paths, three misaligned-theta paths
        for width, off in ((w4, 0), (w4 + 1, 0), (w4 + 2, 0), (w4 + 3, 0), (w4, 1), (w4, 2), (w4, 3)):
            wide = torch.full((k, width), NAN, device=dev)
            wide[:, :n] = st
            buf, th = _views(n, off)
            th.copy_(torch.from_numpy(theta0))
            ops._ext.require().fedavg_apply(th, wide, wt, server_lr)
            torch.cuda.synchronize()
            assert_bits(_np(th), want, f"fedavg_apply lr {server_lr} width {width} theta+{off}")
            assert torch.isnan(buf[:off]).all() and torch.isnan(buf[off + n:]).all()
            del wide


@gpu
@pytest.mark.parametrize("n", [1, 255, 256, 257, 4097])
@pytest.mark.parametrize("rows", [1, 32, 256])
def test_bias_sgd_from_partials_bits(n, rows):
    g = np.random.default_rng(n * 3 + rows)
    part = g.standard_normal((rows, n)).astype(F32)
    gsum = np.zeros(n, F32)
    for r in range(rows):
        gsum = gsum + part[r]                                           # fp32 adds in row order
    assert (np.abs(gsum - part.astype(F64).sum(0)) <= rows * U * np.abs(part.astype(F64)).sum(0)).all()
    n_bias = max(1, n - 3) if n > 1 else 1
    b0 = g.standard_normal(n_bias).astype(F32)
    bias = torch.from_numpy(b0).to(_dev())
    lr = 0.37
    got = ops.bias_sgd_from_partials(bias, torch.from_numpy(part).to(_dev()), lr)
    assert_bits(_np(got), gsum, "bias gradient")
    assert_bits(_np(bias), fmaf_exact(-F32(lr), gsum[:n_bias], b0), "bias step")
    assert_bits(_np(ops.bias_sgd_from_partials(None, torch.from_numpy(part).to(_dev()), lr)), gsum, "gradient only")


def _bf16_specials():
    v = np.array([0.0, -0.0, 1e-45, -1e-45, 1e-39, -5.9e-39, 1.17549435e-38, INF, -INF, NAN, 3.4e38, -3.4e38, 1.0, -1.0],
                 F32)
    # round-half-even ties: low 16 bits exactly 0x8000 on an even and an odd bf16, and one bit either side
    hi = np.array([0x3F80, 0x3F81, 0x4049, 0xC04A, 0x0001, 0x7F7F], np.uint32) << 16
    ties = np.concatenate([hi | 0x8000, hi | 0x7FFF, hi | 0x8001]).view(F32)
    return np.concatenate([v, ties])


@gpu
@pytest.mark.parametrize("n", [1, 3, 5, 4099, VEC_WRAP + 5])
def test_fp32_to_bf16_bits(n):
    g = np.random.default_rng(n + 5)
    with np.errstate(over="ignore"):                       # (a few overflow to +-inf: they belong to the test)
        x = (g.standard_normal(n) * np.exp(g.uniform(-90, 88, n))).astype(F32)
    sp = _bf16_specials()
    x[: min(n, sp.size)] = sp[: min(n, sp.size)]
    want = torch.from_numpy(x).to(torch.bfloat16)
    for off in (0, 1, 2, 3):
        buf, v = _views(n, off)
        v.copy_(torch.from_numpy(x))
        got = ops.fp32_to_bf16(v).cpu()
        nan = torch.isnan(want)
        assert torch.equal(torch.isnan(got), nan)
        assert torch.equal(got[~nan].view(torch.int16), want[~nan].view(torch.int16)), f"offset {off}"


@gpu
@pytest.mark.parametrize("shape", [(1, 1), (1, 1000), (1000, 1), (33, 65), (1025, 31), (32, 32), (64, 96)])
def test_transpose_bf16_bits(shape):
    g = np.random.default_rng(shape[0] * 1000 + shape[1])
    x = torch.from_numpy(g.standard_normal(shape).astype(F32)).to(torch.bfloat16)
    flat = x.view(-1)
    sp = torch.from_numpy(_bf16_specials()).to(torch.bfloat16)
    flat[: min(flat.numel(), sp.numel())] = sp[: min(flat.numel(), sp.numel())]
    got = ops.transpose_bf16(x.to(_dev())).cpu()
    assert torch.equal(got.view(torch.int16), x.t().contiguous().view(torch.int16))    # bits, NaN payloads included


@gpu
@pytest.mark.parametrize("n", [1, 2, 3, 2 ** 16, 2 ** 16 + 1, 10 ** 6 + 7])
def test_feistel_permutation_bijection(n):
    rows = max(2, -(-(SCALAR_WRAP + 1000) // n))
    seed = 0x1234_5678_9ABC
    got = ops.device_permutation(n, rows, seed, _dev())
    assert got.shape == (rows, n)
    srt = torch.sort(got, dim=1).values
    assert torch.equal(srt, torch.arange(n, dtype=torch.int32, device=_dev()).expand(rows, n))
    host = ops._ext.require().feistel_permutation(n, rows, seed, torch.device("cpu"))
    assert torch.equal(got.cpu(), host)
    if n > 100:
        assert not torch.equal(got[0], got[1])


# ---- losses and eval against float64 -------------------------------------------------------------------------------
def _bce_terms(logp, log1mp, t):
    return -(t * _bce_floor(logp) + (1 - t) * _bce_floor(log1mp))


def _sigmoid_f32(e):
    """the kernel's p = 1 / (1 + e) in correctly rounded fp32 steps"""
    with np.errstate(over="ignore"):
        e32 = np.asarray(e, F64).astype(F32)
    return F32(1) / (F32(1) + e32)


def bce_model(z, t):
    """float64 BCE of the kernel's fp32 sigmoid, and an interval that holds what the GPU may return per element:
    __expf(-z) is within expf_rel of exp(-z); 1 + e and 1 / q are IEEE-rounded (monotone), so p lies between the fp32
    sigmoid of the two ends of that range; __logf / log1pf then add logf_abs / log1pf_abs"""
    z64 = z.astype(F64)
    with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
        e = np.exp(-z64)
        E = expf_rel(-z64) + 2 * U
        p_mid = _sigmoid_f32(e)
        p_hi = _sigmoid_f32(e * (1 - E))
        p_lo = _sigmoid_f32(e * (1 + E))
        lp_mid, l1p_mid = np.log(p_mid.astype(F64)), np.log1p(-p_mid.astype(F64))
        lp_lo = np.log(p_lo.astype(F64)) - logf_abs(p_lo)
        lp_hi = np.log(p_hi.astype(F64)) + logf_abs(p_hi)
        l1p_lo = np.log1p(-p_hi.astype(F64)) - log1pf_abs(np.log1p(-p_hi.astype(F64)))
        l1p_hi = np.log1p(-p_lo.astype(F64)) + log1pf_abs(np.log1p(-p_lo.astype(F64)))
    ref = _bce_terms(lp_mid, l1p_mid, t)
    lo = _bce_terms(lp_hi, l1p_hi, t)          # the term is decreasing in both logs
    hi = _bce_terms(lp_lo, l1p_lo, t)
    return ref, lo, hi, p_lo, p_hi


def _check_sum(name, got, ref_terms, lo_terms, hi_terms, scale, rel):
    """got = scale * sum(terms) up to the per-term intervals and `rel` * scale * sum(|terms|) of summation error"""
    if np.isnan(ref_terms).any():
        assert math.isnan(got), f"{name}: a NaN term must give a NaN loss, got {got}"
        return
    ref = ref_terms.sum() * scale
    s_err = rel * np.abs(ref_terms).sum() * scale
    below, above = (ref - lo_terms.sum() * scale) + s_err, (hi_terms.sum() * scale - ref) + s_err
    err = got - ref
    bound = above if err >= 0 else below
    assert abs(err) <= bound, f"{name}: {got} vs float64 {ref}, error {err:.3g} outside the bound {bound:.3g}"
    _record(name, abs(err) / bound if bound > 0 else 0.0)


_Z_SPECIAL = np.array([0.0, 1e-8, -1e-8, 15, -15, 20, -20, 88, -88, 89, -89, 1e4, -1e4, INF, -INF], F32)


@gpu
@pytest.mark.parametrize("n", [1, len(_Z_SPECIAL), 1000, SCALAR_WRAP + 7, 3 * SCALAR_WRAP + 1])
@pytest.mark.parametrize("kind", ["normal", "confident", "nan"])
def test_sigmoid_bce_error_model(n, kind):
    g = np.random.default_rng(n + len(kind))
    z = (g.standard_normal(n) * 4).astype(F32)
    t = (g.random(n) > 0.5).astype(F32)
    if kind == "confident":                         # confident, mostly right: p -> 1 where t = 1
        z = (g.uniform(5, 30, n) * (2 * t - 1)).astype(F32)
        t[::97] = 1 - t[::97]
    k = min(n, _Z_SPECIAL.size)
    z[:k] = _Z_SPECIAL[:k]
    if kind == "nan":
        z[n // 2] = NAN
    loss, dz = ops.sigmoid_bce(torch.from_numpy(z).to(_dev()), torch.from_numpy(t).to(_dev()))
    ref, lo, hi, p_lo, p_hi = bce_model(z, t.astype(F64))
    blocks = _grid(n)
    _check_sum("sigmoid_bce loss", float(loss), ref, lo, hi, 1.0 / n, sum_rel(-(-n // (blocks * THREADS)), 8, blocks))
    # dz = (p - t) * (1 / n): IEEE steps, monotone in p -> an exact interval
    inv_n = F32(1) / F32(n)
    d_lo, d_hi = (p_lo - t) * inv_n, (p_hi - t) * inv_n
    dzn = _np(dz).reshape(-1)
    nan = np.isnan(z)
    assert np.array_equal(np.isnan(dzn), nan)
    ok = (dzn >= d_lo) & (dzn <= d_hi)
    assert ok[~nan].all(), f"dz outside its interval at {np.flatnonzero(~ok & ~nan)[:5]}"


def eval_model(p, t):
    p64 = p.astype(F64)
    with np.errstate(divide="ignore", invalid="ignore"):
        lp, l1p = np.log(p64), np.log1p(-p64)
    ref = _bce_terms(lp, l1p, t)
    lo = _bce_terms(lp + logf_abs(p64), l1p + log1pf_abs(l1p), t)
    hi = _bce_terms(lp - logf_abs(p64), l1p - log1pf_abs(l1p), t)
    return ref, lo, hi


_P_SPECIAL = np.array([0.0, 1.0, 0.5, 1 - 2 ** -24, 2 ** -126, 1e-45, 0.5 - 2 ** -25, 0.5 + 2 ** -24], F32)


@gpu
@pytest.mark.parametrize("n", [1, _P_SPECIAL.size * 2, 999, SCALAR_WRAP + 7, 3 * SCALAR_WRAP + 1])
@pytest.mark.parametrize("kind", ["uniform", "confident", "nan"])
def test_eval_binary_error_model(n, kind):
    g = np.random.default_rng(n + 3 * len(kind))
    t = (g.random(n) > 0.5).astype(F32)
    if kind == "confident":     # confident correct predictions: log p ~ -1e-4 .. -6e-8, where __logf's bound is absolute
        q = (1 - np.exp(g.uniform(-16.6, -9, n))).astype(F32)
        p = np.where(t == 1, q, 1 - q).astype(F32)
    else:
        p = g.random(n).astype(F32)
    k = min(n, 2 * _P_SPECIAL.size)
    p[:k] = np.tile(_P_SPECIAL, 2)[:k]
    t[:k] = np.repeat([1.0, 0.0], _P_SPECIAL.size)[:k]
    if kind == "nan":
        p[-1] = NAN
    loss, correct = ops.eval_binary(torch.from_numpy(p).to(_dev()), torch.from_numpy(t).to(_dev()))
    want_correct = int((torch.round(torch.from_numpy(p)) == torch.from_numpy(t)).sum())
    assert int(correct) == want_correct
    ref, lo, hi = eval_model(p, t.astype(F64))
    blocks = _grid(n)
    _check_sum("eval_binary loss", float(loss), ref, lo, hi, 1.0, sum_rel(-(-n // (blocks * THREADS)), 8, blocks))
    if kind == "nan":
        assert math.isnan(float(R.eval_binary(torch.from_numpy(p), torch.from_numpy(t))[0]))


@gpu
@pytest.mark.parametrize("n", [1, 1000, SCALAR_WRAP + 7, 3 * SCALAR_WRAP + 1])
@pytest.mark.parametrize("mean", [False, True])
@pytest.mark.parametrize("mag", [1e-15, 1.0, 1e3])
def test_sse_error_model(n, mean, mag):
    g = np.random.default_rng(n)
    out = (g.standard_normal(n) * 10 * min(1.0, mag * 1e4)).astype(F32)     # tiny differences between tiny values
    y = (out + g.standard_normal(n) * mag).astype(F32)
    loss, dz = ops.sse_loss(torch.from_numpy(out).to(_dev()).view(n, 1), torch.from_numpy(y).to(_dev()).view(n, 1), mean=mean)
    scale = F32(1.0 / n) if mean else F32(1.0)
    d = out - y                                                            # fp32, as the kernel rounds it
    assert_bits(_np(dz).reshape(-1), F32(2) * d * scale, "sse dz")
    exact = (out.astype(F64) - y.astype(F64)) ** 2
    blocks = _grid(n)
    slack = exact * 3 * U + 2.0 ** -149                                    # the rounded difference, squared
    _check_sum("sse loss", float(loss), exact, exact - slack, exact + slack, F64(scale),
               sum_rel(-(-n // (blocks * THREADS)), 8, blocks))


def xent_model(z32, labels):
    """float64 softmax cross-entropy of fp32 logits, and per-row loss / per-element gradient bounds for the kernel:
    s = sum_c __expf(z_c - m) (the fp32 difference is the kernel's own), each term within expf_rel, summed per lane
    (ceil(cols / 32) adds) and over 5 shuffle levels; loss = (__logf(s) + m) - z_label with logf_abs at s; gradient
    (__expf(z - m) / s - [c == label]) / rows"""
    rows, cols = z32.shape
    m32 = z32.max(1, keepdims=True)
    with np.errstate(invalid="ignore", over="ignore"):
        x = (z32 - m32).astype(F64)
        t = np.exp(x)
        s = t.sum(1, keepdims=True)
        sig = (t * expf_rel(x)).sum(1, keepdims=True) / s + (-(-cols // 32) + 5) * U
        p = t / s
        zl = z32[np.arange(rows), labels].astype(F64)
        logs = np.log(s[:, 0])
        loss = logs + m32[:, 0].astype(F64) - zl
        loss_b = logf_abs(s[:, 0]) + sig[:, 0] / (1 - sig[:, 0]) + 2 * U * (np.abs(logs + m32[:, 0]) + np.abs(loss))
        onehot = np.zeros_like(p)
        onehot[np.arange(rows), labels] = 1
        grad = (p - onehot) / rows
        grad_b = (p * (expf_rel(x) + sig + 3 * U) + 3 * U * np.abs(p - onehot)) / rows + 2.0 ** -148
    return loss, loss_b, grad, grad_b


def _logits(rows, cols, kind, g):
    labels = g.integers(0, cols, rows)
    labels[0], labels[-1] = 0, cols - 1
    if kind == "flat":
        z = g.standard_normal((rows, cols)) * 1e-3
    elif kind == "confident":                     # the label's logit 10..40 above the rest: s -> 1, loss ~ s - 1
        z = g.standard_normal((rows, cols))
        z[np.arange(rows), labels] = z.max(1) + g.uniform(10, 40, rows)
    else:                                          # "specials": -inf / -1e30 away from the label, large magnitudes
        z = g.standard_normal((rows, cols)) * 30
        if cols > 1:
            other = (labels + 1) % cols
            z[np.arange(0, rows, 3), other[::3]] = -np.inf
            z[np.arange(1, rows, 3), other[1::3]] = -1e30
    return z.astype(F32), labels


@gpu
@pytest.mark.parametrize("cols", [1, 2, 31, 32, 33, 100, 1024, 1500])
@pytest.mark.parametrize("kind", ["flat", "confident", "specials"])
def test_softmax_xent_error_model(cols, kind):
    rows = 2 * ROW_WRAP + 5 if cols <= 100 else 300
    g = np.random.default_rng(cols * 10 + len(kind))
    z, labels = _logits(rows, cols, kind, g)
    lab = torch.from_numpy(labels).to(_dev())
    for bf16_in in (False, True):
        zin = torch.from_numpy(z).to(_dev())
        if bf16_in:
            zin = zin.to(torch.bfloat16)
        zq = zin.float().cpu().numpy()
        loss, dl = ops.softmax_xent(zin, lab)
        lref, lb, gref, gb = xent_model(zq, labels)
        warps = min(-(-rows // 8), GRID_CAP) * 8
        _check_sum("softmax_xent loss", float(loss), lref, lref - lb, lref + lb, 1.0 / rows,
                   sum_rel(-(-rows // warps), 5, warps))
        err = np.abs(_np(dl).astype(F64) - gref)
        assert (err <= gb).all(), f"gradient error {err.max():.3g} over its bound at {np.unravel_index(np.argmax(err - gb), err.shape)}"
        _record("softmax_xent grad", (err / gb).max())
        # the bf16 gradient is the fp32 one rounded to bf16 (same kernel, same g)
        lb16, dl16 = ops.softmax_xent(zin, lab, bf16_grad=True)
        assert dl16.dtype == torch.bfloat16
        assert torch.equal(dl16.view(torch.int16), dl.to(torch.bfloat16).view(torch.int16))
        assert float(lb16) == pytest.approx(float(loss), rel=1e-5, abs=1e-9)      # (atomics: any order)


@gpu
def test_softmax_xent_nonfinite_rows():
    """+inf logits give a non-finite loss on both sides; a label at -inf gives +inf; an all -inf row gives NaN"""
    z = np.array([[1.0, INF, 0.0], [0.0, 1.0, -INF], [-INF, -INF, -INF], [3.0, 2.0, 1.0]], F32)
    for labels, finite in (([0, 0, 0, 0], False), ([0, 2, 0, 0], False), ([1, 0, 0, 0], False)):
        lab = torch.tensor(labels)
        loss, _ = ops.softmax_xent(torch.from_numpy(z).to(_dev()), lab.to(_dev()))
        ref, _ = R.softmax_xent(torch.from_numpy(z), lab)
        assert not math.isfinite(float(loss)) and not math.isfinite(float(ref))
    loss, _ = ops.softmax_xent(torch.from_numpy(z[1:2]).to(_dev()), torch.tensor([2], device=_dev()))
    assert float(loss) == INF


@gpu
@pytest.mark.parametrize("rows", [1, 31, 32, 33, 1024, 1025])
@pytest.mark.parametrize("cols", [1, 32, 33, 128])
@pytest.mark.parametrize("bf16_in", [False, True])
def test_softmax_xent_head_error_model(rows, cols, bf16_in):
    g = np.random.default_rng(rows * 1000 + cols + bf16_in)
    z, labels = _logits(rows, cols, "confident" if rows % 2 else "specials", g)
    ld = cols + 5
    dev = _dev()
    big = torch.full((rows + 2, ld), 123.0, device=dev)
    big[:rows, :cols] = torch.from_numpy(z).to(dev)
    if bf16_in:
        big = big.to(torch.bfloat16)
    zq = big[:rows, :cols].float().cpu().numpy()
    lab = torch.from_numpy(np.concatenate([labels, [0, 0]])).to(dev)
    from colearn_federated_learning_b200.ops import conv as C
    outs = []
    for _ in range(2):
        d32 = torch.full((rows + 2, ld + 1), 7.0, device=dev)
        d16 = torch.full((rows + 2, ld + 3), 7.0, device=dev, dtype=torch.bfloat16)
        db = torch.full((ld,), 7.0, device=dev)
        loss = C.softmax_xent_head(big, lab, rows, cols, dl_bf16=d16, db=db, dl_f32=d32)
        outs.append((loss.clone(), d32.clone(), d16.clone(), db.clone()))
    assert all(torch.equal(a, b) for a, b in zip(outs[0], outs[1]))                       # fixed summation order
    loss, d32, d16, db = outs[0]
    assert (d32[rows:] == 7).all() and (d32[:, cols:] == 7).all() and (d16[rows:] == 7).all() and (d16[:, cols:] == 7).all()
    assert (db[cols:] == 7).all()
    assert torch.equal(d16[:rows, :cols].view(torch.int16), d32[:rows, :cols].to(torch.bfloat16).view(torch.int16))
    lref, lb, gref, gb = xent_model(zq, labels)
    nw = min(rows, 32)
    _check_sum("softmax_xent_head loss", float(loss), lref, lref - lb, lref + lb, 1.0 / rows, sum_rel(-(-rows // nw), 5, nw))
    got = _np(d32[:rows, :cols]).astype(F64)
    err = np.abs(got - gref)
    assert (err <= gb).all(), f"gradient error {err.max():.3g} over its bound"
    _record("softmax_xent_head grad", (err / gb).max())
    # the bias gradient: column sums of the kernel's own fp32 gradient, per warp then over the warps
    want_db = got.sum(0)
    db_b = sum_rel(-(-rows // nw), 0, nw) * np.abs(got).sum(0) + 2.0 ** -149
    assert (np.abs(_np(db[:cols]) - want_db) <= db_b).all()


@gpu
@pytest.mark.parametrize("cols", [1, 2, 31, 32, 33, 1000])
def test_argmax_rows_matches_torch(cols):
    rows = 2 * ROW_WRAP + 9 if cols < 1000 else ROW_WRAP + 9
    g = np.random.default_rng(cols)
    x = g.standard_normal((rows, cols)).astype(F32)
    if cols > 2:
        x[::5, 1] = x[::5].max(1)                          # ties with a later maximum
    sp = _argmax_special_rows(cols)
    x[: sp.shape[0]] = sp
    x[-sp.shape[0]:] = sp                                  # and again in the second grid-stride pass
    xt = torch.from_numpy(x)
    got = ops.argmax_rows(xt.to(_dev())).cpu()
    assert torch.equal(got, xt.argmax(1, keepdim=True))


def _minmax_emulated(x):
    """the kernel's own fp32 arithmetic, NaN left out of the column's min / max: (x - lo) * (1 / rng)"""
    with np.errstate(invalid="ignore"):
        lo = np.nanmin(np.where(np.isnan(x), np.inf, x), 0).astype(F32)
        hi = np.nanmax(np.where(np.isnan(x), -np.inf, x), 0).astype(F32)
    rng = hi - lo
    rng = np.where(rng == 0, F32(1), rng).astype(F32)
    return (x - lo) * (F32(1) / rng), lo, hi


@gpu
@pytest.mark.parametrize("rows", [1, 1023, 1024, 1025, 100_000])
@pytest.mark.parametrize("cols", [1, 10, 77])
def test_minmax_scale_bits_and_float64(rows, cols):
    g = np.random.default_rng(rows + cols)
    mags = np.exp(g.uniform(-30, 30, cols))
    x = (g.standard_normal((rows, cols)) * mags + g.standard_normal(cols) * mags * 3).astype(F32)
    if cols > 1:
        x[:, 1] = F32(2.5)                                 # a constant column
    if cols > 2:
        x[:, 2] = (1e6 + g.random(rows)).astype(F32)       # large offset, small spread
    if cols > 3 and rows > 1:
        x[rows // 2, 3] = NAN
    got = _np(ops.minmax_scale(torch.from_numpy(x).to(_dev())))
    want, lo, hi = _minmax_emulated(x)
    assert_bits(got, want, "minmax_scale")
    fin = ~np.isnan(x)
    rng = (hi - lo).astype(F64)                            # the column's fp32 range, as the kernel has it
    exact = np.where(rng == 0, 0.0, (x.astype(F64) - lo) / np.where(rng == 0, 1, rng))
    assert (ulps(got[fin], exact[fin]) <= 2).all()         # x - lo, 1 / rng and the product: three roundings
    assert (got[x == lo] == 0).all()
    if cols > 1:
        assert (got[:, 1] == 0).all()
    cpu = _np(ops.minmax_scale(torch.from_numpy(x)))
    assert np.array_equal(np.isnan(cpu), np.isnan(x)) and (ulps(cpu[fin], got[fin]) <= 2).all()


# ---- end to end: fl.evaluate on the GPU vs a float64 evaluation on the CPU ----------------------------------------
@gpu
@pytest.mark.parametrize("ctor", [FFNN, MLP])
@pytest.mark.parametrize("nan_bias", [False, True])
def test_evaluate_end_to_end(ctor, nan_bias):
    from colearn_federated_learning_b200.fl.evaluate import evaluate, forward_flat, predict
    torch.manual_seed(11)
    model = ctor()
    spec = model.spec
    n = 100_003
    x = torch.rand(n, spec.dims[0]) * 2
    xent = spec.default_loss == "xent"
    y = (torch.randint(0, spec.dims[-1], (n, 1)).float() if xent else (torch.rand(n, 1) > 0.5).float())
    flat = flatten_params(model).clone()
    j = spec.dims[-1] - 1
    if nan_bias:
        flat[spec.offsets()[-1][1] + j] = NAN
    dev = _dev()
    res = evaluate(model, x.to(dev), y.to(dev), flat.to(dev), verbose=False)
    out = forward_flat(model, flat.to(dev), x.to(dev)).float().cpu()
    out64, _ = R.mlp_forward(flat.double(), spec.dims, x.double(), spec.out_activation)
    if xent:
        lab = y.view(-1).long()
        loss64 = float(R.loss_and_dz(out64, lab.view(-1, 1).double(), "xent", "none")[0])
        pred = predict(model, x.to(dev), flat.to(dev)).cpu()
        assert torch.equal(pred, out.argmax(1, keepdim=True))
        if nan_bias:
            assert (pred == j).all()
        assert res["correct"] == int((pred.view(-1) == lab).sum())
        top2 = out64.topk(2, dim=1).values if spec.dims[-1] > 1 else None
        near = int(((top2[:, 0] - top2[:, 1]).abs() < 1e-4).sum()) if top2 is not None else 0
        assert abs(res["correct"] - int((out64.argmax(1) == lab).sum())) <= near
        lref, lb, _, _ = xent_model(out.numpy(), lab.numpy())
        if not nan_bias:
            warps = min(-(-n // 8), GRID_CAP) * 8
            _check_sum("evaluate xent loss", res["loss"], lref, lref - lb, lref + lb, 1.0 / n, sum_rel(-(-n // warps), 5, warps))
    else:
        p = out.view(-1).numpy()
        t = y.view(-1).numpy()
        loss64 = float(R.eval_binary(out64.view(-1), y.view(-1).double())[0]) / n
        assert res["correct"] == int((torch.round(out.view(-1)) == y.view(-1)).sum())
        near = int(((out64.view(-1) - 0.5).abs() < 1e-4).sum())
        assert abs(res["correct"] - int((torch.round(out64.view(-1)) == y.view(-1).double()).sum())) <= near
        if not nan_bias:
            ref, lo, hi = eval_model(p, t.astype(F64))
            _check_sum("evaluate bce loss", res["loss"] * n, ref, lo, hi, 1.0, sum_rel(1, 8, _grid(n)))
    if nan_bias:
        assert math.isnan(res["loss"]) and math.isnan(loss64)
    else:
        assert abs(res["loss"] - loss64) <= 1e-4 * abs(loss64) + 1e-6
