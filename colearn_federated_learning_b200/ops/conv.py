"""NHWC convolution / BatchNorm / pooling ops around the wgmma GEMM (csrc/convnet.cu, SURVEY K17).

Activations are NHWC flattened to a row-major bf16 matrix ``[M = N*H*W, C]``; a convolution is
``im2col`` (``k = (kh, kw, c)``) followed by ``ops.gemm_bf16``; the other ops are BatchNorm (training
statistics / apply with fused residual + ReLU / backward), max / average pooling and the weight (un)packing
between torch's ``[Cout, Cin, KH, KW]`` arena layout and the padded ``[Cout_pad, K_pad]`` GEMM layout.

Three backends share one signature per op:

* CUDA tensors  -> the hand-written sm_90a kernels (``_colearn_C``; mandatory on a GPU box);
* CPU tensors   -> the pure-PyTorch definitions in this file (the oracle the kernels are tested against);
* CPU tensors inside :func:`emulated` -> ``_colearn_emul``: the *kernel bodies themselves* (``csrc/conv_ops.cuh``)
  compiled for the host, so the index arithmetic of every kernel is exercised by the CPU test-suite.

All ops write into caller-provided buffers (the trainer owns every buffer, so a step is allocation-free and
CUDA-graph capturable).  The PyTorch definitions round to whatever dtype the destination buffer has (``copy_``):
bf16 buffers reproduce the kernels' rounding points, fp32 buffers give an exact oracle for the orchestration.
"""
from __future__ import annotations

import contextlib
import glob
import importlib.util
import os
from typing import List, Optional, Sequence

import torch
import torch.nn.functional as F

from . import _ext

_EMUL = {"on": False, "mod": None, "simt": None}
_HERE = os.path.dirname(os.path.abspath(__file__))


def load_emulator(build_if_missing: bool = True):
    """Import (building on first use) the CPU emulator of the conv kernels."""
    if _EMUL["mod"] is None:
        hits = sorted(glob.glob(os.path.join(_HERE, "_colearn_emul*.so")))
        if not hits and build_if_missing:
            from . import build
            hits = [build.build_emul()]
        if not hits:
            raise FileNotFoundError("_colearn_emul*.so not built (python -m colearn_federated_learning_b200.ops.build --emul)")
        spec = importlib.util.spec_from_file_location("_colearn_emul", hits[0])
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)  # type: ignore[union-attr]
        _EMUL["mod"] = mod
    return _EMUL["mod"]


@contextlib.contextmanager
def emulated():
    """Route CPU tensors through the host build of the kernel bodies instead of the PyTorch definitions."""
    load_emulator()
    prev, _EMUL["on"] = _EMUL["on"], True
    try:
        yield
    finally:
        _EMUL["on"] = prev


def load_simt(build_if_missing: bool = True):
    """Import (building on first use) ``_colearn_simt``: the conv kernels' CUDA *launchers and kernels* (csrc/convnet.cu)
    compiled for the CPU through csrc/host_shim.h — one OS thread per CUDA thread (tests only)."""
    if _EMUL["simt"] is None:
        hits = sorted(glob.glob(os.path.join(_HERE, "_colearn_simt*.so")))
        if build_if_missing:
            from . import build
            hits = [build.build_simt_emul()]           # no-op when the objects are current
        if not hits:
            raise FileNotFoundError("_colearn_simt*.so not built (python -m colearn_federated_learning_b200.ops.build --simt)")
        spec = importlib.util.spec_from_file_location("_colearn_simt", hits[0])
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)  # type: ignore[union-attr]
        _EMUL["simt"] = mod
    return _EMUL["simt"]


@contextlib.contextmanager
def simt():
    """Route CPU tensors through the SIMT-on-CPU build of the kernels themselves (grid mapping, shared-memory phases,
    atomics included) instead of the PyTorch definitions."""
    mod = load_simt()
    prev_on, prev_mod = _EMUL["on"], _EMUL["mod"]
    _EMUL["on"], _EMUL["mod"] = True, mod
    try:
        yield
    finally:
        _EMUL["on"], _EMUL["mod"] = prev_on, prev_mod


def _native(t: torch.Tensor):
    """The compiled module that should handle ``t`` (None -> use the PyTorch definition)."""
    if t.is_cuda:
        return _ext.require()
    return _EMUL["mod"] if _EMUL["on"] else None


def softmax_xent_head(logits: torch.Tensor, labels: torch.Tensor, rows: int, cols: int, dl_bf16: Optional[torch.Tensor] = None,
                      db: Optional[torch.Tensor] = None, dl_f32: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Loss head of the GEMM-shaped trainers in one launch (``softmax_xent_head_kernel``): mean softmax cross-entropy of
    ``logits[:rows, :cols]`` (a padded fp32 / bf16 matrix); ``dL/dlogits`` goes straight into ``dl_bf16[:rows, :cols]`` (the
    padded operand of the backward GEMMs) and / or ``dl_f32``, its column sums (the head's bias gradient) into ``db[:cols]``.
    One block with a fixed summation order: bit-reproducible.  ``cols <= 128``."""
    mod = _native(logits)
    labels = labels.reshape(-1)
    if labels.dtype != torch.long:
        labels = labels.long()
    if mod is not None and hasattr(mod, "softmax_xent_head"):
        return mod.softmax_xent_head(logits, labels.contiguous(), int(rows), int(cols), dl_f32, dl_bf16, db)
    from . import reference
    loss, g = reference.softmax_xent(logits[:rows, :cols].float(), labels[:rows])
    if dl_f32 is not None:
        dl_f32[:rows, :cols].copy_(g)
    if dl_bf16 is not None:
        dl_bf16[:rows, :cols].copy_(g)
    if db is not None:
        db[:cols].copy_(g.sum(0))
    return loss


def out_size(h: int, k: int, stride: int, pad: int) -> int:
    return (h + 2 * pad - k) // stride + 1


def nhwc_view(act: torch.Tensor, n: int, h: int, w: int, c: int) -> torch.Tensor:
    """Logical ``[N, C, H, W]`` (strided) view of an NHWC activation matrix ``[>= N*H*W, C]``."""
    return act[: n * h * w].view(n, h, w, c).permute(0, 3, 1, 2)


# ----------------------------------------------------------------------------------------------------------
# im2col / col2im
# ----------------------------------------------------------------------------------------------------------
def im2col(x4: torch.Tensor, col: torch.Tensor, kh: int, kw: int, stride: int, pad: int) -> None:
    """``col[m, (kh*KW + kw)*C + c] = x[n, c, oh*stride - pad + kh, ow*stride - pad + kw]`` (zero outside the
    image and in the pad columns).  ``x4``: strided ``[N, C, H, W]`` view, fp32 or bf16; ``col``: bf16
    ``[>= N*OH*OW, K_pad]``."""
    mod = _native(col)
    if mod is not None:
        mod.im2col(x4, col, kh, kw, stride, pad)
        return
    n, c, h, w = x4.shape
    oh, ow = out_size(h, kh, stride, pad), out_size(w, kw, stride, pad)
    cols = F.unfold(x4.float(), (kh, kw), padding=pad, stride=stride)             # [N, C*KH*KW, L], k = (c, kh, kw)
    cols = cols.view(n, c, kh * kw, oh * ow).permute(0, 3, 2, 1).reshape(n * oh * ow, kh * kw * c)
    m, k = cols.shape
    col[:m, :k].copy_(cols)
    col[:m, k:].zero_()


def col2im(dcol: torch.Tensor, dx: torch.Tensor, add: Optional[torch.Tensor], n: int, h: int, w: int, c: int,
           kh: int, kw: int, stride: int, pad: int) -> None:
    """Adjoint of :func:`im2col` as a gather: ``dx[N*H*W, C] = fold(dcol) (+ add)`` (bf16)."""
    mod = _native(dx)
    if mod is not None:
        mod.col2im(dcol, dx, add, n, h, w, c, kh, kw, stride, pad)
        return
    oh, ow = out_size(h, kh, stride, pad), out_size(w, kw, stride, pad)
    m, k = n * oh * ow, kh * kw * c
    d = dcol[:m, :k].float().view(n, oh * ow, kh * kw, c).permute(0, 3, 2, 1).reshape(n, c * kh * kw, oh * ow)
    dx4 = F.fold(d, (h, w), (kh, kw), padding=pad, stride=stride)
    res = dx4.permute(0, 2, 3, 1).reshape(n * h * w, c)
    if add is not None:
        res = res + add[: n * h * w].float()
    dx[: n * h * w].copy_(res)


# ----------------------------------------------------------------------------------------------------------
# BatchNorm (training mode)
# ----------------------------------------------------------------------------------------------------------
def bn_partial_numel(m: int, c: int) -> int:
    """fp32 scratch the BatchNorm reductions need for an ``[m, c]`` input (2 quantities x <= 64 row segments)."""
    rows = max(32, ((m + 63) // 64 + 31) // 32 * 32)
    return 2 * c * ((m + rows - 1) // rows)


def bn_stats(x: torch.Tensor, c: int, partial: torch.Tensor, mean: torch.Tensor, invstd: torch.Tensor,
             running_mean: Optional[torch.Tensor] = None, running_var: Optional[torch.Tensor] = None,
             eps: float = 1e-5, momentum: float = 0.1, counters: Optional[torch.Tensor] = None) -> None:
    """Per-channel batch mean and ``1/sqrt(var + eps)`` (biased variance) of ``x[:, :c]`` (bf16 ``[M, ldx]``);
    running statistics updated in place with torch semantics (unbiased variance, ``momentum``).  ``counters``
    (int32 ``[c/64]``, zero before the first use, self-resetting) selects the single-launch reduction whose last
    block finalises."""
    mod = _native(x)
    if mod is not None:
        mod.bn_stats(x, c, partial, mean, invstd, running_mean, running_var, float(eps), float(momentum), counters)
        return
    xf = x[:, :c].float()
    m = xf.shape[0]
    mu = xf.mean(0)
    var = (xf * xf).mean(0) - mu * mu
    var = var.clamp_min(0)
    mean[:c].copy_(mu)
    invstd[:c].copy_(torch.rsqrt(var + eps))
    if running_mean is not None:
        running_mean[:c].mul_(1 - momentum).add_(momentum * mu)
        running_var[:c].mul_(1 - momentum).add_(momentum * var * (m / max(m - 1, 1)))


def bn_apply(x: torch.Tensor, c: int, mean: torch.Tensor, invstd: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor,
             res: Optional[torch.Tensor], relu: bool, out: torch.Tensor) -> None:
    """``out = relu?((x - mean) * invstd * gamma + beta (+ res))`` → bf16 ``[M, c]``."""
    mod = _native(x)
    if mod is not None:
        mod.bn_apply(x, c, mean, invstd, gamma, beta, res, bool(relu), out)
        return
    m = x.shape[0]
    y = (x[:, :c].float() - mean[:c]) * invstd[:c] * gamma[:c] + beta[:c]
    if res is not None:
        y = y + res[:m].float()
    if relu:
        y = torch.relu(y)
    out[:m].copy_(y)


def bn_backward(x: torch.Tensor, c: int, dy: torch.Tensor, out: Optional[torch.Tensor], mean: torch.Tensor,
                invstd: torch.Tensor, gamma: torch.Tensor, partial: torch.Tensor, dgamma: torch.Tensor, dbeta: torch.Tensor,
                dx: torch.Tensor, g_out: Optional[torch.Tensor] = None, counters: Optional[torch.Tensor] = None) -> None:
    """BatchNorm backward.  With ``out`` (the layer's post-ReLU output) the upstream gradient is masked first
    (``g = dy * (out > 0)``; optionally written to ``g_out`` for the identity branch of a residual block).

    ``dbeta = Σ g``, ``dgamma = Σ g·x̂``, ``dx = γ·invstd·(g − dbeta/M − x̂·dgamma/M)``."""
    mod = _native(x)
    if mod is not None:
        mod.bn_backward(x, c, dy, out, mean, invstd, gamma, partial, dgamma, dbeta, dx, g_out, counters)
        return
    m = x.shape[0]
    g = dy[:m].float()
    if out is not None:
        g = g * (out[:m].float() > 0)
    xh = (x[:, :c].float() - mean[:c]) * invstd[:c]
    db = g.sum(0)
    dg = (g * xh).sum(0)
    dbeta[:c].copy_(db)
    dgamma[:c].copy_(dg)
    dx[:m].copy_(gamma[:c] * invstd[:c] * (g - db / m - xh * dg / m))
    if g_out is not None:
        g_out[:m].copy_(g)


# ----------------------------------------------------------------------------------------------------------
# pooling
# ----------------------------------------------------------------------------------------------------------
def maxpool_fwd(x: torch.Tensor, out: torch.Tensor, idx: torch.Tensor, n: int, h: int, w: int, c: int, kh: int, kw: int,
                stride: int, pad: int) -> None:
    """NHWC max pooling; ``idx`` (uint8) records the window offset ``kh*KW + kw`` of the (first) maximum."""
    mod = _native(x)
    if mod is not None:
        mod.maxpool_fwd(x, out, idx, n, h, w, c, kh, kw, stride, pad)
        return
    oh, ow = out_size(h, kh, stride, pad), out_size(w, kw, stride, pad)
    x4 = nhwc_view(x, n, h, w, c).float()
    y, flat = F.max_pool2d(x4, (kh, kw), stride, pad, return_indices=True)      # flat = ih*W + iw
    ih, iw = flat // w, flat % w
    base_h = (torch.arange(oh) * stride - pad).view(1, 1, oh, 1)
    base_w = (torch.arange(ow) * stride - pad).view(1, 1, 1, ow)
    code = (ih - base_h) * kw + (iw - base_w)
    out[: n * oh * ow].copy_(y.permute(0, 2, 3, 1).reshape(n * oh * ow, c))
    idx[: n * oh * ow].copy_(code.permute(0, 2, 3, 1).reshape(n * oh * ow, c).to(torch.uint8))


def maxpool_bwd(dy: torch.Tensor, idx: torch.Tensor, dx: torch.Tensor, n: int, h: int, w: int, c: int, kh: int, kw: int,
                stride: int, pad: int) -> None:
    mod = _native(dy)
    if mod is not None:
        mod.maxpool_bwd(dy, idx, dx, n, h, w, c, kh, kw, stride, pad)
        return
    oh, ow = out_size(h, kh, stride, pad), out_size(w, kw, stride, pad)
    code = idx[: n * oh * ow].view(n, oh, ow, c).long()
    ih = torch.arange(oh).view(1, oh, 1, 1) * stride - pad + code // kw
    iw = torch.arange(ow).view(1, 1, ow, 1) * stride - pad + code % kw
    nn_ = torch.arange(n).view(n, 1, 1, 1).expand_as(code)
    cc = torch.arange(c).view(1, 1, 1, c).expand_as(code)
    lin = ((nn_ * h + ih) * w + iw) * c + cc
    acc = torch.zeros(n * h * w * c)
    acc.index_add_(0, lin.reshape(-1), dy[: n * oh * ow].float().reshape(-1))
    dx[: n * h * w].copy_(acc.view(n * h * w, c))


def avgpool_fwd(x: torch.Tensor, out: torch.Tensor, n: int, hw: int, c: int) -> None:
    mod = _native(x)
    if mod is not None:
        mod.avgpool_fwd(x, out, n, hw, c)
        return
    out[:n].copy_(x[: n * hw].float().view(n, hw, c).mean(1))


def avgpool_bwd(dy: torch.Tensor, dx: torch.Tensor, n: int, hw: int, c: int) -> None:
    mod = _native(dy)
    if mod is not None:
        mod.avgpool_bwd(dy, dx, n, hw, c)
        return
    dx[: n * hw].copy_((dy[:n].float() / hw).view(n, 1, c).expand(n, hw, c).reshape(n * hw, c))


# ----------------------------------------------------------------------------------------------------------
# weight packing: flat arena (torch layouts) <-> padded GEMM layouts
# ----------------------------------------------------------------------------------------------------------
class PackEntry:
    """One ``[rows, cols]`` matrix of the flat arena and its padded slot in the packed buffers.  ``channels > 0``
    marks a conv weight ``[Cout, Cin, KH, KW]`` whose columns are permuted to ``(kh, kw, c)``."""

    def __init__(self, name: str, src_off: int, rows: int, cols: int, rows_pad: int, cols_pad: int, channels: int = 0,
                 khw: int = 1) -> None:
        self.name, self.src_off, self.rows, self.cols = name, int(src_off), int(rows), int(cols)
        self.rows_pad, self.cols_pad, self.channels, self.khw = int(rows_pad), int(cols_pad), int(channels), int(khw)
        self.dst_off = 0

    @property
    def numel_pad(self) -> int:
        return self.rows_pad * self.cols_pad


class PackPlan:
    """Descriptor table for :func:`pack_params` (one launch moves every layer)."""

    def __init__(self, entries: Sequence[PackEntry], device) -> None:
        self.entries: List[PackEntry] = list(entries)
        off = 0
        for e in self.entries:
            e.dst_off = off
            off += e.numel_pad
        self.total = off
        self.device = torch.device(device)
        self._descs: Optional[torch.Tensor] = None

    def view(self, buf: torch.Tensor, e: PackEntry) -> torch.Tensor:
        return buf[e.dst_off:e.dst_off + e.numel_pad].view(e.rows_pad, e.cols_pad)

    def descs(self, mod) -> torch.Tensor:
        if self._descs is None:
            raw = b"".join(mod.make_pack_desc(e.src_off, e.dst_off, e.rows, e.cols, e.rows_pad, e.cols_pad, e.channels, e.khw)
                           for e in self.entries)
            self._descs = torch.frombuffer(bytearray(raw), dtype=torch.uint8).to(self.device)
        return self._descs


def pack_params(arena: torch.Tensor, packed_f32: torch.Tensor, packed_bf16: Optional[torch.Tensor], plan: PackPlan,
                unpack: bool = False) -> None:
    """``unpack=False``: arena → ``packed_f32`` (+ bf16 copy), permuted and zero padded.  ``unpack=True``:
    ``packed_f32`` → arena (valid region only)."""
    mod = _native(arena)
    if mod is not None:
        mod.pack_params(arena, packed_f32, packed_bf16, plan.descs(mod), len(plan.entries), bool(unpack))
        return
    for e in plan.entries:
        src = arena[e.src_off:e.src_off + e.rows * e.cols].view(e.rows, e.cols)
        dst = plan.view(packed_f32, e)
        if e.channels > 0:   # [rows, C, KHW] <-> [rows, KHW, C]
            if unpack:
                src.copy_(dst[: e.rows, : e.cols].reshape(e.rows, e.khw, e.channels).permute(0, 2, 1).reshape(e.rows, e.cols))
            else:
                dst.zero_()
                dst[: e.rows, : e.cols].copy_(src.view(e.rows, e.channels, e.khw).permute(0, 2, 1).reshape(e.rows, e.cols))
        else:
            if unpack:
                src.copy_(dst[: e.rows, : e.cols])
            else:
                dst.zero_()
                dst[: e.rows, : e.cols].copy_(src)
    if not unpack and packed_bf16 is not None:
        packed_bf16.copy_(packed_f32)


# ----------------------------------------------------------------------------------------------------------
# split-K GEMM: reduction of the partial accumulators + the epilogue the un-split GEMM would have fused
# ----------------------------------------------------------------------------------------------------------
def splitk_reduce(part: torch.Tensor, splits: int, numel: int, *, master: Optional[torch.Tensor] = None, lr: float = 0.0,
                  shadow: Optional[torch.Tensor] = None, out_bf16: Optional[torch.Tensor] = None) -> None:
    """Sum the ``splits`` fp32 partials ``part[s, numel]`` a split-K ``ops.gemm_bf16`` left behind (in slice order)
    and finish the GEMM: with ``master`` the fused SGD step of a wgrad (``master -= lr·Σ``, ``shadow`` = the bf16
    copy the next forward reads), otherwise ``out_bf16 = Σ`` rounded to the buffer's dtype."""
    assert (master is None) != (out_bf16 is None)
    mod = _native(part)
    if mod is not None:
        mod.splitk_reduce(part, int(splits), int(numel), master, float(lr), shadow, out_bf16)
        return
    p = part[: splits * numel].view(splits, numel)
    acc = p[0].clone()
    for s in range(1, splits):
        acc += p[s]
    if master is not None:
        m = master.view(-1)[:numel]
        m.sub_(lr * acc)
        if shadow is not None:
            shadow.view(-1)[:numel].copy_(m)
    else:
        out_bf16.view(-1)[:numel].copy_(acc)


# ----------------------------------------------------------------------------------------------------------
# implicit-GEMM convolution (stride 1): the activation is read through a 4-D TMA tensor map, no col matrix
# ----------------------------------------------------------------------------------------------------------
def implicit_ok(h: int, w: int, c: int, stride: int, n: int = 128) -> bool:
    """Geometries the implicit path covers: stride 1, 64-channel blocks, images of 1 / 4 / 16 / 64 pixels (a GEMM tile
    of 128 pixels — 64 for the wgrad's reduction blocks — is then a box of whole images)."""
    return stride == 1 and c % 64 == 0 and h * w in (1, 4, 16, 64) and (n * h * w) % 128 == 0


def conv_gemm(kind: str, act: torch.Tensor, other: torch.Tensor, n: int, h: int, w: int, c: int, kh: int, kw: int, pad: int, *,
              out_bf16: Optional[torch.Tensor] = None, addend: Optional[torch.Tensor] = None, rows_per_tap: int = 0,
              m_pad: int = 0, k_pad: int = 0, w_packed: bool = False, sgd_master: Optional[torch.Tensor] = None, sgd_lr: float = 0.0,
              sgd_shadow: Optional[torch.Tensor] = None, split_k: int = 0, split_out: Optional[torch.Tensor] = None) -> None:
    """The three GEMMs of a stride-1 convolution with the NHWC activation ``act`` (``[n*h*w, c]`` bf16) as an implicit
    operand (``csrc/conv_ops.cuh``: ``ConvAddr``; boxes of whole images through a 4-D tensor map, TMA zero fill = the
    padding).  ``kind``:

    * ``"fwd"``   ``out[p, co] = Σ act[p + tap − pad, ·]·other[co, tap·c + ·]`` — ``other`` = packed weights ``[Cout_pad, K_pad]``
    * ``"dgrad"`` ``out[p, ci] = Σ act[p + pad − tap, ·]·other[tap·rows_per_tap + ci, ·] (+ addend)`` — ``act`` = dz
      ``[pixels, c = Cout]``, ``other`` = ``Wᵀ`` ``[K_pad, Cout]``, ``rows_per_tap`` = Cin; with ``w_packed=True`` ``other`` is
      the packed ``Wp[Cout_pad, K_pad]`` itself (MN-major B operand: no ``Wᵀ`` copy to keep in step with the updates)
    * ``"wgrad"`` ``dW[co, tap·c + ·] = Σ_p other[p, co]·act[p + tap − pad, ·]`` — ``other`` = dz ``[pixels, Cout]``; the
      result (``[m_pad, k_pad]``, K padding = zeros) goes through the fused SGD epilogue or the split-K partials.

    CPU tensors use the PyTorch definitions (``im2col`` / ``col2im`` + the reference GEMM), CUDA the wgmma kernel."""
    from .linear import gemm_bf16
    m = n * h * w
    taps = kh * kw
    simt_mod = _EMUL["mod"] if (_EMUL["on"] and not act.is_cuda and hasattr(_EMUL["mod"], "gemm_tcgen05")) else None
    if act.is_cuda or simt_mod is not None:
        mod = _ext.require() if act.is_cuda else simt_mod
        if kind == "wgrad":
            assert m_pad > 0 and k_pad >= taps * c
            geom = [2, 0, c, kh, kw, pad, h, w, n, 0, m_pad, k_pad, m, 0]
        elif kind == "fwd":
            geom = [1, 0, c, kh, kw, pad, h, w, n, 0, m, out_bf16.shape[1] if out_bf16 is not None else other.shape[0], taps * c, 0]
        else:
            geom = [1, 1, c, kh, kw, pad, h, w, n, rows_per_tap, m, rows_per_tap, taps * c, 1 if w_packed else 0]
        if simt_mod is not None:   # the kernel source on the functional wgmma / TMA model (csrc/gemm_host_model.h)
            mod.gemm_tcgen05(act, other, None, False, None, out_bf16, None, None, sgd_master, float(sgd_lr), sgd_shadow, None, None,
                             0, int(split_k or 0), split_out, 0, False, addend, geom, [])
            return
        mod.gemm_tcgen05(act, other, None, False, None, out_bf16, None, None, sgd_master, float(sgd_lr), sgd_shadow, None, None,
                         0, 0, 1, 0, 0, 0, 0, int(split_k or 0), split_out, 0, False, addend, geom, [])
        return
    # --- definitions --------------------------------------------------------------------------------------------
    x4 = nhwc_view(act, n, h, w, c)
    k = taps * c
    if kind == "fwd":
        col = torch.zeros(m, k, dtype=act.dtype)
        im2col(x4, col, kh, kw, 1, pad)
        if split_k and split_k > 1:     # slices of the implicit K loop: k-blocks of 64 over (tap, c)
            nn_ = other.shape[0]
            part = split_out[: split_k * m * nn_].view(split_k, m, nn_)
            nkb = k // 64
            for s_ in range(split_k):
                lo, hi = nkb * s_ // split_k * 64, nkb * (s_ + 1) // split_k * 64
                part[s_].copy_(col[:, lo:hi].float() @ other[:, lo:hi].float().t())
            return
        out_bf16.copy_(col.float() @ other[:, :k].float().t())
    elif kind == "dgrad":
        cin = rows_per_tap
        wt = (other[:c, : taps * cin].t() if w_packed else other[: taps * cin, :c]).float()   # [taps*cin, cout]
        dcol = act[:m].float() @ wt.t()                                     # [m, taps*cin], k = (tap, ci)
        dx = torch.zeros(m, cin, dtype=out_bf16.dtype)
        col2im(dcol.to(out_bf16.dtype), dx, addend, n, h, w, cin, kh, kw, 1, pad)
        out_bf16[:m].copy_(dx)
    elif kind == "wgrad":
        col = torch.zeros(m, k, dtype=act.dtype)
        im2col(x4, col, kh, kw, 1, pad)
        assert m_pad > 0 and k_pad >= k
        colp = torch.zeros(m, k_pad, dtype=act.dtype)
        colp[:, :k] = col
        gemm_bf16(other, colp, mn_m=m_pad, sgd_master=sgd_master, sgd_lr=sgd_lr, sgd_shadow=sgd_shadow, split_k=split_k,
                  split_out=split_out)
    else:
        raise ValueError(kind)
