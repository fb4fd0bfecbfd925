"""Local training of ResNet-18 on this repo's own kernels (BASELINE config 4, SURVEY K17).

Every convolution is ``im2col`` + the wgmma GEMM (``ops.gemm_bf16``) in its three roles,

    forward   z[M, Cout]      = col[M, K]      · Wp[Cout, K]ᵀ                      (M = N·OH·OW, k = (kh, kw, c))
    dgrad     dcol[M, K]      = dz[M, Cout]    · (Wpᵀ)[K, Cout]ᵀ   → col2im gather → dx
    wgrad     Wp[Cout, K]    -= lr · dzᵀ[Cout, M] · colᵀ[K, M]ᵀ    (SGD fused in the GEMM epilogue: fp32 master +
                                                                    bf16 shadow refreshed, dW never materialised)

with NHWC bf16 activations, so the GEMM output *is* the next layer's activation matrix.  BatchNorm (training
statistics, apply + residual + ReLU, backward with the ReLU mask folded in), max / average pooling and the
weight (un)packing are the kernels of ``ops/csrc/convnet.cu``; the loss is ``ops.softmax_xent`` and the small
parameters (γ, β, fc bias) take one flat ``ops.sgd_step``.  During a fit the *packed* fp32 weights
(``[Cout_pad, K_pad]``, what the wgrad epilogue updates) are the master copy; ``load`` packs them from the flat
arena FedAvg averages and ``store`` unpacks them back, once per fit each.

Numerics follow the autocast-bf16 torch path this replaces (bf16 operands / activations, fp32 accumulation,
fp32 statistics and parameters).  No reference counterpart: the reference has no conv nets (SURVEY §2.5 K17).
"""
from __future__ import annotations

import os
import weakref
from typing import Dict, List, Optional, Tuple

import torch
import torch.nn as nn

from .. import ops
from ..models.registry import param_layout
from ..models.resnet import BasicBlock, ResNet18
from ..ops import conv as C

BF = torch.bfloat16
PAD = 128

# Step schedule.  Every entry is a re-scheduling / operand-layout choice with the same mathematical result.  The values
# below are the schedule the ResNet-18 step ships with; 0 everywhere is the round-1 schedule (explicit im2col, K-major operands from transposed copies, one
# stream).  The environment (COLEARN_CONV_<NAME>=<int>) overrides in both directions, constructor arguments override
# the environment.
SCHEDULE_DEFAULTS = {
    "STREAMS": 1,     # 1: wgrad chains on a second stream inside the step graph
    "SHADOW_T": 0,    # 1: W^T written by the wgrad epilogue instead of a transpose launch (moot with DGRAD_KN: no W^T exists)
    "FUSED_BN": 1,    # 1: BatchNorm reduction + finalize in one launch
    "SPLITK": 1,      # 1: split-K for the skinny wgrad GEMMs, 2: also the layer4 forwards
    "WGRAD_MN": 1,    # 1: wgrad GEMMs read dz / col in place (MN-major operands)
    "DGRAD_KN": 1,    # 1: dgrad GEMMs read the packed weights (MN-major B), no W^T copies
    "IMPLICIT": 2,    # 1: implicit-GEMM forward + dgrad for the stride-1 3x3 convs, 2: wgrad too
}


def schedule_flag(name: str) -> int:
    v = os.environ.get("COLEARN_CONV_" + name, "").strip()
    return int(v) if v else SCHEDULE_DEFAULTS[name]


def _pad(n: int, m: int = PAD) -> int:
    return (n + m - 1) // m * m


class _Conv:
    """Geometry + buffers of one convolution (+ the BatchNorm that follows it)."""

    def __init__(self, name: str, mod: nn.Conv2d, bn_name: str, bn: nn.BatchNorm2d, n: int, h: int, w: int) -> None:
        self.name, self.bn_name = name, bn_name
        self.cin, self.cout = mod.in_channels, mod.out_channels
        self.k, self.stride, self.pad = mod.kernel_size[0], mod.stride[0], mod.padding[0]
        self.n, self.h, self.w = n, h, w
        self.oh, self.ow = C.out_size(h, self.k, self.stride, self.pad), C.out_size(w, self.k, self.stride, self.pad)
        self.m_in, self.m = n * h * w, n * self.oh * self.ow
        self.K = self.k * self.k * self.cin
        self.K_pad, self.cout_pad = _pad(self.K), _pad(self.cout)
        self.eps, self.momentum = bn.eps, (0.1 if bn.momentum is None else bn.momentum)
        self.entry: Optional[C.PackEntry] = None
        self.implicit = False                          # implicit-GEMM schedule (4-D TMA boxes instead of im2col / col2im)
        self.x_in: Optional[torch.Tensor] = None       # the layer's input activation matrix [m_in, cin] (implicit wgrad)

    def alloc(self, dev, act_dtype: torch.dtype = BF) -> None:
        z = lambda *s, dt=act_dtype: torch.zeros(*s, device=dev, dtype=dt)  # noqa: E731
        self.col = z(self.m, self.K_pad)              # saved for the wgrad
        self.z = z(self.m, self.cout_pad)             # conv output (pre-BN), pitch cout_pad
        self.out = z(self.m, self.cout)               # post BN (+res) (+ReLU) activation
        self.mean = z(self.cout, dt=torch.float32)
        self.invstd = z(self.cout, dt=torch.float32)
        self.rm = self.rv = None                      # running statistics: views handed out by the trainer
        self.wT = z(self.K_pad, self.cout)            # bf16 Wpᵀ (valid rows only) for the dgrad
        self.dz = z(self.m, self.cout)                # gradient w.r.t. the conv output


class _Block:
    def __init__(self, c1: _Conv, c2: _Conv, ds: Optional[_Conv]) -> None:
        self.c1, self.c2, self.ds = c1, c2, ds


class ConvNetTrainer:
    """SGD steps of :class:`~colearn_federated_learning_b200.models.resnet.ResNet18` on a flat fp32 arena."""

    _cache: Dict[Tuple, "ConvNetTrainer"] = {}

    # -- construction --------------------------------------------------------------------------------------
    @staticmethod
    def supports(model: nn.Module, cfg, x: torch.Tensor) -> bool:
        return (isinstance(model, ResNet18) and cfg.loss == "xent" and cfg.batch_size % 128 == 0 and x.dim() == 4
                and x.shape[1] == model.conv1.in_channels and x.shape[0] >= cfg.batch_size
                and x.shape[0] % cfg.batch_size == 0          # a ragged last batch stays on the autograd path
                and x.shape[2] >= 32 and x.shape[3] >= 32)

    @classmethod
    def cached(cls, model: ResNet18, flat: torch.Tensor, batch_size: int, hw: Tuple[int, int]) -> "ConvNetTrainer":
        key = (id(model), flat.data_ptr(), str(flat.device), batch_size, tuple(hw))
        tr = cls._cache.get(key)
        if tr is not None and tr._model_ref() is not model:      # id() of a collected module got recycled
            tr = None
        if tr is None:
            if len(cls._cache) > 2:
                cls._cache.clear()
            tr = cls._cache[key] = cls(model, flat.device, batch_size, hw)
            tr._model_ref = weakref.ref(model)
            tr.bind_buffers(model)
        return tr

    def __init__(self, model: ResNet18, device, batch_size: int, hw: Tuple[int, int] = (32, 32),
                 act_dtype: torch.dtype = BF, split_k: Optional[bool] = None, wgrad_mn: Optional[bool] = None,
                 dgrad_kn: Optional[bool] = None, implicit: Optional[int] = None) -> None:
        """``act_dtype=torch.float32`` (CPU only) keeps every buffer in fp32: the PyTorch definitions of the ops then
        make the whole step an exact oracle for the orchestration (tests compare it with autograd).  ``split_k``
        (default: ``COLEARN_CONV_SPLITK=1``) runs the skinny GEMMs — the wgrads of the stem / layer1 / layer2 (1-5 output
        tiles, reductions over up to 32 768 pixels) and the forwards of layer3 / layer4 — in split-K mode, see
        :meth:`_pick_split` (``1`` / ``True``: wgrads only, ``2``: forwards too).  ``wgrad_mn`` (default:
        ``COLEARN_CONV_WGRAD_MN=1``) feeds the wgrad GEMMs ``dz`` and ``col`` as they are (MN-major wgmma operands,
        reduction over rows) instead of transposing both first; ``dgrad_kn`` (``COLEARN_CONV_DGRAD_KN=1``) lets the
        dgrad GEMMs read the packed weights ``Wp[Cout, K]`` as an MN-major B operand, so no ``Wᵀ`` copy is kept.
        ``implicit`` (``COLEARN_CONV_IMPLICIT=1|2``): the stride-1 3x3 convolutions whose images have 1-64 pixels (13 of
        the 20) run as implicit GEMMs — forward and dgrad read x / dz through 4-D TMA boxes (``ops.conv.conv_gemm``;
        level 2: the wgrad too, which needs the MN-major path), so ``col`` / ``dcol`` / ``col2im`` disappear."""
        assert batch_size % 128 == 0, "the GEMM tiles need batch_size % 128 == 0"
        assert act_dtype == BF or torch.device(device).type == "cpu", "the kernels are bf16"
        self.dev, self.B, self.dt = torch.device(device), batch_size, act_dtype
        self.num_classes = model.fc.out_features
        dev, B = self.dev, batch_size
        layout = {name: (off, shape) for name, shape, off, _ in param_layout(model)}
        self.n_params = sum(n for _, _, _, n in param_layout(model))

        # ---- geometry -------------------------------------------------------------------------------------
        h, w = hw
        self.stem = _Conv("conv1", model.conv1, "bn1", model.bn1, B, h, w)
        h, w = self.stem.oh, self.stem.ow
        self.pool_in = (h, w)
        self.pool_k, self.pool_s, self.pool_p = 3, 2, 1
        h, w = C.out_size(h, 3, 2, 1), C.out_size(w, 3, 2, 1)
        self.pool_out = (h, w)
        self.blocks: List[_Block] = []
        for li in range(1, 5):
            for bi, blk in enumerate(getattr(model, f"layer{li}")):
                assert isinstance(blk, BasicBlock)
                p = f"layer{li}.{bi}"
                c1 = _Conv(f"{p}.conv1", blk.conv1, f"{p}.bn1", blk.bn1, B, h, w)
                c2 = _Conv(f"{p}.conv2", blk.conv2, f"{p}.bn2", blk.bn2, B, c1.oh, c1.ow)
                ds = None
                if blk.downsample is not None:
                    ds = _Conv(f"{p}.downsample.0", blk.downsample[0], f"{p}.downsample.1", blk.downsample[1], B, h, w)
                self.blocks.append(_Block(c1, c2, ds))
                h, w = c2.oh, c2.ow
        self.final_hw = h * w
        self.feat_dim = self.blocks[-1].c2.cout
        self.convs: List[_Conv] = [self.stem] + [c for b in self.blocks for c in ((b.c1, b.c2, b.ds) if b.ds else (b.c1, b.c2))]

        # ---- packed big parameters: conv weights + fc weight ([rows_pad, cols_pad], GEMM layout) ---------------
        entries = []
        for cv in self.convs:
            off, _ = layout[cv.name + ".weight"]
            cv.entry = C.PackEntry(cv.name + ".weight", off, cv.cout, cv.K, cv.cout_pad, cv.K_pad, cv.cin, cv.k * cv.k)
            entries.append(cv.entry)
        off, _ = layout["fc.weight"]
        self.nc_pad = _pad(self.num_classes)
        self.fc_entry = C.PackEntry("fc.weight", off, self.num_classes, self.feat_dim, self.nc_pad, _pad(self.feat_dim))
        entries.append(self.fc_entry)
        self.big = C.PackPlan(entries, dev)
        self.mpk = torch.zeros(self.big.total, device=dev)                       # fp32 master (during a fit)
        self.wpk = torch.zeros(self.big.total, device=dev, dtype=act_dtype)      # bf16 shadow (GEMM operand)

        # ---- packed small parameters: gamma / beta of every BatchNorm, fc bias (padded) -----------------------
        small = []
        for cv in self.convs:
            for leaf in ("weight", "bias"):
                off, _ = layout[f"{cv.bn_name}.{leaf}"]
                small.append(C.PackEntry(f"{cv.bn_name}.{leaf}", off, 1, cv.cout, 1, cv.cout))
        off, _ = layout["fc.bias"]
        small.append(C.PackEntry("fc.bias", off, 1, self.num_classes, 1, self.nc_pad))
        self.small = C.PackPlan(small, dev)
        self.spk = torch.zeros(self.small.total, device=dev)
        self.gsp = torch.zeros(self.small.total, device=dev)
        self._small_by_name = {e.name: e for e in self.small.entries}

        # ---- buffers ------------------------------------------------------------------------------------------
        for cv in self.convs:
            cv.alloc(dev, act_dtype)
        # BatchNorm buffers of every layer in three flat tensors; bind_buffers() can alias the module's buffers onto
        # them so the kernels update the module in place and a fit needs no buffer copies
        tot_c = sum(cv.cout for cv in self.convs)
        self.running_mean = torch.zeros(tot_c, device=dev)
        self.running_var = torch.ones(tot_c, device=dev)
        self.batches_tracked = torch.zeros(len(self.convs), device=dev, dtype=torch.long)
        off = 0
        for cv in self.convs:
            cv.rm, cv.rv = self.running_mean[off:off + cv.cout], self.running_var[off:off + cv.cout]
            off += cv.cout
        self._bound: Optional[nn.Module] = None
        self._model_ref = weakref.ref(model)
        # opt-in: wgrad chains on a second stream, see _conv_bwd
        self._side = torch.cuda.Stream(self.dev) if (self.dev.type == "cuda" and schedule_flag("STREAMS")) else None
        self._fuse_shadow_t = bool(schedule_flag("SHADOW_T"))
        # opt-in: BatchNorm reduction + finalize in one launch (ticket counter, last block finalises)
        self.bn_counters = (torch.zeros(max(cv.cout for cv in self.convs) // 64, device=dev, dtype=torch.int32)
                            if schedule_flag("FUSED_BN") and act_dtype == BF else None)
        self._graph = None
        self._graph_key = None
        z = lambda *s, dt=act_dtype: torch.zeros(*s, device=dev, dtype=dt)  # noqa: E731
        # opt-in: split-K for the GEMMs with too few output tiles to fill the SMs
        # opt-in: wgrad GEMMs on MN-major operands — no dz^T / col^T transposes
        self._wgrad_mn = bool(schedule_flag("WGRAD_MN")) if wgrad_mn is None else bool(wgrad_mn)
        # opt-in: dgrad GEMMs against the packed weights themselves (MN-major B operand) — no W^T copies to refresh
        self._dgrad_kn = bool(schedule_flag("DGRAD_KN")) if dgrad_kn is None else bool(dgrad_kn)
        # opt-in: implicit GEMM for the stride-1 3x3 convolutions (1: forward + dgrad, 2: wgrad too)
        self._implicit = schedule_flag("IMPLICIT") if implicit is None else int(implicit)
        for cv in self.convs:
            cv.implicit = (self._implicit > 0 and cv.k == 3 and cv.pad == 1 and cv.cout % 64 == 0
                           and C.implicit_ok(cv.h, cv.w, cv.cin, cv.stride, B))
        # COLEARN_CONV_SPLITK=1: wgrads only; =2: forwards too
        self._splitk = schedule_flag("SPLITK") if split_k is None else int(split_k)
        for cv in self.convs:
            cv.s_fwd = self._pick_split(cv.m, cv.cout_pad, cv.K_pad, min_slices=8) if self._splitk >= 2 else 1
            cv.s_wgrad = self._pick_split(cv.cout_pad, cv.K_pad, cv.m, min_slices=4) if self._splitk >= 1 else 1
            if cv.implicit and cv.h * cv.w == 1:
                cv.s_fwd = 1       # 1x1 images: the implicit GEMM walks the centre tap only (K = C), nothing left to split
        # fp32 partial accumulators [S, M, N]; forward and wgrad have their own (the wgrad chains may run on a side stream)
        self.kpart_f = z(max([cv.s_fwd * cv.m * cv.cout_pad for cv in self.convs if cv.s_fwd > 1] or [4]), dt=torch.float32)
        self.kpart_w = z(max([cv.s_wgrad * cv.cout_pad * cv.K_pad for cv in self.convs if cv.s_wgrad > 1] or [4]), dt=torch.float32)
        max_colT = max(cv.m * cv.K_pad for cv in self.convs)
        max_dzT = max(cv.m * cv.cout_pad for cv in self.convs)
        self.colT = z(max_colT)                        # scratch: colᵀ of the layer whose wgrad runs
        self.dcol = z(max_colT)                        # scratch: dgrad GEMM output
        self.dzT = z(max_dzT)                          # scratch: dzᵀ padded to cout_pad rows
        self.partial = z(max(C.bn_partial_numel(cv.m, cv.cout) for cv in self.convs), dt=torch.float32)
        m_pool = B * self.pool_out[0] * self.pool_out[1]
        self.pool_y = z(m_pool, self.stem.cout)
        self.pool_idx = torch.zeros(m_pool, self.stem.cout, device=dev, dtype=torch.uint8)
        self.d_pool = z(m_pool, self.stem.cout)        # gradient w.r.t. the pooled stem output
        self.d_stem = z(self.stem.m, self.stem.cout)   # gradient w.r.t. the stem activation
        for b in self.blocks:
            b.g = z(b.c2.m, b.c2.cout)                 # masked gradient at the block output (identity branch)
            b.d_mid = z(b.c1.m, b.c1.cout)             # gradient w.r.t. relu(bn1(conv1))
            b.d_in = z(b.c1.m_in, b.c1.cin)            # gradient w.r.t. the block input
            b.d_skip = z(b.c1.m_in, b.c1.cin) if b.ds else None
        self.feat = z(B, self.feat_dim)
        self.featT = z(self.feat_dim, B)
        self.d_feat = z(B, self.feat_dim)
        self.d_last = z(self.blocks[-1].c2.m, self.feat_dim)
        self.logits = z(B, self.nc_pad, dt=torch.float32)
        self.dlog = z(B, self.nc_pad)
        self.dlogT = z(self.nc_pad, B)
        self.fc_wT = z(self.feat_dim, self.nc_pad)
        self.launches = 0
        self.steps_done = 0                            # since the last store() (BatchNorm num_batches_tracked)
        self.steps_total = 0

    @staticmethod
    def _pick_split(m: int, n: int, k: int, min_slices: int = 2, sms: int = 148) -> int:
        """Number of K slices for a ``[m, n] = [m, k]·[n, k]ᵀ`` GEMM: 1 when the output already has enough tiles
        (128 x 256 when ``n % 256 == 0``, else 128 x 128) to occupy the machine, otherwise as many slices as it takes to
        give every SM a work unit while each slice keeps >= 8 k-blocks of 64 (a pipeline's worth); fewer than
        ``min_slices`` slices are not worth the extra reduction launch.  E.g. batch 128, 32x32 images: stem wgrad
        128x256x32768 -> 1 tile x 64 slices; layer1 wgrad 128x640x8192 -> 5 tiles x 16."""
        tiles = (m // 128) * (n // (256 if n % 256 == 0 else 128))
        if tiles >= sms // 2:
            return 1
        s = min((k // 64) // 8, -(-sms // tiles))
        return s if s >= max(2, min_slices) else 1

    def _needs_wT(self, cv: _Conv) -> bool:
        """A bf16 ``Wᵀ`` copy is the dgrad's K-major B operand; ``dgrad_kn`` (explicit and implicit schedule alike) reads
        the packed weights instead."""
        return not self._dgrad_kn

    def _gemm_fwd(self, cv: _Conv) -> None:
        """``cv.z = cv.col · Wpᵀ`` (bf16), split-K when the layer has few output tiles."""
        if cv.s_fwd > 1:
            ops.gemm_bf16(cv.col, self._w(cv.entry), split_k=cv.s_fwd, split_out=self.kpart_f)
            C.splitk_reduce(self.kpart_f, cv.s_fwd, cv.m * cv.cout_pad, out_bf16=cv.z)
            self.launches += 1
        else:
            ops.gemm_bf16(cv.col, self._w(cv.entry), out_bf16=cv.z)

    # -- parameter views ------------------------------------------------------------------------------------------
    def _w(self, e: C.PackEntry) -> torch.Tensor:
        return self.big.view(self.wpk, e)

    def _m(self, e: C.PackEntry) -> torch.Tensor:
        return self.big.view(self.mpk, e)

    def _s(self, name: str, buf: Optional[torch.Tensor] = None) -> torch.Tensor:
        e = self._small_by_name[name]
        return (self.spk if buf is None else buf)[e.dst_off:e.dst_off + e.numel_pad]

    def bind_buffers(self, model: ResNet18) -> bool:
        """Alias the module's BatchNorm buffers onto this trainer's flat statistics tensors (zero-copy, like
        ``alias_params_to_arena`` for parameters).  Only possible when the module lives on the trainer's device."""
        mods = dict(model.named_modules())
        if any(mods[cv.bn_name].running_mean.device != self.running_mean.device for cv in self.convs):
            return False
        with torch.no_grad():
            for i, cv in enumerate(self.convs):
                bn = mods[cv.bn_name]
                cv.rm.copy_(bn.running_mean)
                cv.rv.copy_(bn.running_var)
                self.batches_tracked[i] = bn.num_batches_tracked
                bn.running_mean.data, bn.running_var.data = cv.rm, cv.rv
                bn.num_batches_tracked.data = self.batches_tracked[i]
        self._bound = model
        return True

    def load(self, flat: torch.Tensor, model: Optional[ResNet18] = None) -> None:
        """Flat arena (and the module's BatchNorm buffers, unless bound) → packed device state."""
        C.pack_params(flat, self.mpk, self.wpk, self.big)
        C.pack_params(flat, self.spk, None, self.small)
        for cv in self.convs:
            if self._needs_wT(cv):
                ops.transpose_bf16(self._w(cv.entry)[: cv.cout], cv.wT)
        ops.transpose_bf16(self._w(self.fc_entry), self.fc_wT)
        if model is not None and model is not self._bound:
            mods = dict(model.named_modules())
            for cv in self.convs:
                bn = mods[cv.bn_name]
                cv.rm.copy_(bn.running_mean)
                cv.rv.copy_(bn.running_var)
        self.launches += 3 + sum(1 for cv in self.convs if self._needs_wT(cv))

    def store(self, flat: torch.Tensor, model: Optional[ResNet18] = None) -> None:
        """Packed device state → flat arena (and the module's BatchNorm buffers, unless bound)."""
        C.pack_params(flat, self.mpk, None, self.big, unpack=True)
        C.pack_params(flat, self.spk, None, self.small, unpack=True)
        if model is not None and model is self._bound:
            self.batches_tracked += self.steps_done
        elif model is not None:
            mods = dict(model.named_modules())
            with torch.no_grad():
                for cv in self.convs:
                    bn = mods[cv.bn_name]
                    bn.running_mean.copy_(cv.rm)
                    bn.running_var.copy_(cv.rv)
                    bn.num_batches_tracked += self.steps_done
        self.steps_done = 0
        self.launches += 3

    # -- forward ------------------------------------------------------------------------------------------------------
    def _conv_fwd(self, cv: _Conv, x4: torch.Tensor, xmat: Optional[torch.Tensor]) -> None:
        """``cv.z`` = the convolution of the layer input (``x4``: strided NCHW view; ``xmat``: the same data as the NHWC
        matrix ``[m_in, cin]`` when the producer was one of this trainer's kernels)."""
        if cv.implicit and xmat is not None:
            cv.x_in = xmat
            if cv.s_fwd > 1:
                C.conv_gemm("fwd", xmat, self._w(cv.entry), cv.n, cv.h, cv.w, cv.cin, cv.k, cv.k, cv.pad, split_k=cv.s_fwd,
                            split_out=self.kpart_f)
                C.splitk_reduce(self.kpart_f, cv.s_fwd, cv.m * cv.cout_pad, out_bf16=cv.z)
                self.launches += 1
            else:
                C.conv_gemm("fwd", xmat, self._w(cv.entry), cv.n, cv.h, cv.w, cv.cin, cv.k, cv.k, cv.pad, out_bf16=cv.z)
            self.launches -= 1                         # no im2col launch on this path (callers count 5 per conv)
            return
        C.im2col(x4, cv.col, cv.k, cv.k, cv.stride, cv.pad)
        self._gemm_fwd(cv)

    def _conv_bn(self, cv: _Conv, x4: torch.Tensor, res: Optional[torch.Tensor], relu: bool,
                 xmat: Optional[torch.Tensor] = None) -> torch.Tensor:
        self._conv_fwd(cv, x4, xmat)
        C.bn_stats(cv.z, cv.cout, self.partial, cv.mean, cv.invstd, cv.rm, cv.rv, cv.eps, cv.momentum, self.bn_counters)
        C.bn_apply(cv.z, cv.cout, cv.mean, cv.invstd, self._s(cv.bn_name + ".weight"), self._s(cv.bn_name + ".bias"),
                   res, relu, cv.out)
        self.launches += 5
        return cv.out

    def forward(self, xb: torch.Tensor, labels: torch.Tensor) -> torch.Tensor:
        """Training-mode forward of one batch (``xb``: ``[B, Cin, H, W]`` fp32 or bf16); returns the mean loss."""
        B = self.B
        st = self.stem
        a = self._conv_bn(st, xb, None, True)
        C.maxpool_fwd(a, self.pool_y, self.pool_idx, B, st.oh, st.ow, st.cout, self.pool_k, self.pool_k, self.pool_s, self.pool_p)
        a = self.pool_y
        for b in self.blocks:
            c1, c2 = b.c1, b.c2
            x4 = C.nhwc_view(a, B, c1.h, c1.w, c1.cin)
            identity = a if b.ds is None else self._conv_bn(b.ds, x4, None, False)
            mid = self._conv_bn(c1, x4, None, True, xmat=a)
            a = self._conv_bn(c2, C.nhwc_view(mid, B, c2.h, c2.w, c2.cin), identity, True, xmat=mid)
        C.avgpool_fwd(a, self.feat, B, self.final_hw, self.feat_dim)
        ops.gemm_bf16(self.feat, self._w(self.fc_entry), bias=self._s("fc.bias"), out_f32=self.logits)
        # loss head: logits (padded fp32) -> dL/dlogits in the padded bf16 operand of the fc backward GEMMs + fc.bias gradient + loss
        loss = C.softmax_xent_head(self.logits, labels, B, self.num_classes, dl_bf16=self.dlog, db=self._s("fc.bias", self.gsp))
        self.launches += 8
        return loss

    # -- inference (eval mode: BatchNorm uses the running statistics) -------------------------------------------------------
    @torch.no_grad()
    def infer(self, x: torch.Tensor) -> torch.Tensor:
        """Eval-mode logits ``[n, num_classes]`` (fp32) for ``x`` ``[n, Cin, H, W]`` with the currently loaded
        parameters (call :meth:`load` first).  Runs in chunks of the trainer's batch size; the last chunk is zero
        padded (eval-mode BatchNorm has no cross-sample coupling, so padding rows do not disturb real rows)."""
        B, n = self.B, x.shape[0]
        inv_all = torch.rsqrt(self.running_var + self.stem.eps)
        out = torch.empty(n, self.num_classes, device=self.dev)
        off, invs = 0, {}
        for cv in self.convs:
            invs[cv.name] = inv_all[off:off + cv.cout]
            off += cv.cout

        def conv_bn(cv: _Conv, x4, res, relu, xmat=None):
            self._conv_fwd(cv, x4, xmat)
            C.bn_apply(cv.z, cv.cout, cv.rm, invs[cv.name], self._s(cv.bn_name + ".weight"), self._s(cv.bn_name + ".bias"),
                       res, relu, cv.out)
            return cv.out

        for lo in range(0, n, B):
            xb = x[lo:lo + B]
            if xb.shape[0] < B:
                xb = torch.cat([xb, xb.new_zeros(B - xb.shape[0], *xb.shape[1:])])
            st = self.stem
            a = conv_bn(st, xb.contiguous(), None, True)
            C.maxpool_fwd(a, self.pool_y, self.pool_idx, B, st.oh, st.ow, st.cout, self.pool_k, self.pool_k, self.pool_s, self.pool_p)
            a = self.pool_y
            for b in self.blocks:
                c1, c2 = b.c1, b.c2
                x4 = C.nhwc_view(a, B, c1.h, c1.w, c1.cin)
                identity = a if b.ds is None else conv_bn(b.ds, x4, None, False)
                mid = conv_bn(c1, x4, None, True, xmat=a)
                a = conv_bn(c2, C.nhwc_view(mid, B, c2.h, c2.w, c2.cin), identity, True, xmat=mid)
            C.avgpool_fwd(a, self.feat, B, self.final_hw, self.feat_dim)
            ops.gemm_bf16(self.feat, self._w(self.fc_entry), bias=self._s("fc.bias"), out_f32=self.logits)
            k = min(B, n - lo)
            out[lo:lo + k].copy_(self.logits[:k, : self.num_classes])
        return out

    # -- backward (+ SGD) ---------------------------------------------------------------------------------------------------
    def _bn_bwd(self, cv: _Conv, dy: torch.Tensor, masked: bool, g_out: Optional[torch.Tensor]) -> None:
        C.bn_backward(cv.z, cv.cout, dy, cv.out if masked else None, cv.mean, cv.invstd, self._s(cv.bn_name + ".weight"),
                      self.partial, self._s(cv.bn_name + ".weight", self.gsp), self._s(cv.bn_name + ".bias", self.gsp),
                      cv.dz, g_out, self.bn_counters)
        self.launches += 3

    def _dgrad(self, cv: _Conv, dx: torch.Tensor, add: Optional[torch.Tensor]) -> None:
        if cv.implicit and cv.x_in is not None:
            # dx[p, ci] = Σ_(tap, co) dz[p + pad − tap, co]·Wᵀ[(tap, ci), co] (+ the identity branch's gradient): dz boxes
            # through the 4-D map, no dcol, no col2im
            if self._dgrad_kn:     # ... against the packed weights themselves (MN-major B), no W^T copy
                C.conv_gemm("dgrad", cv.dz, self._w(cv.entry), cv.n, cv.oh, cv.ow, cv.cout, cv.k, cv.k, cv.pad, out_bf16=dx,
                            addend=add, rows_per_tap=cv.cin, w_packed=True)
            else:
                C.conv_gemm("dgrad", cv.dz, cv.wT, cv.n, cv.oh, cv.ow, cv.cout, cv.k, cv.k, cv.pad, out_bf16=dx, addend=add,
                            rows_per_tap=cv.cin)
            self.launches += 1
            return
        dcol = self.dcol[: cv.m * cv.K_pad].view(cv.m, cv.K_pad)
        if self._dgrad_kn:   # dcol[pixel, k] = Σ_co dz[pixel, co]·Wp[co, k]: B is the packed weight matrix itself
            ops.gemm_bf16(cv.dz, self._w(cv.entry), b_kn=True, out_bf16=dcol)
        else:
            ops.gemm_bf16(cv.dz, cv.wT, out_bf16=dcol)
        C.col2im(dcol, dx, add, cv.n, cv.h, cv.w, cv.cin, cv.k, cv.k, cv.stride, cv.pad)
        self.launches += 2

    def _wgrad(self, cv: _Conv, lr: float, shadow_t: bool = False) -> None:
        if cv.implicit and cv.x_in is not None:
            if self._implicit >= 2:
                # dW[co, (tap, c)] = Σ_p dz[p, co]·x[p + tap − pad, c]: dz MN-major, x through 64-pixel boxes — no col at all
                if cv.s_wgrad > 1:
                    C.conv_gemm("wgrad", cv.x_in, cv.dz, cv.n, cv.h, cv.w, cv.cin, cv.k, cv.k, cv.pad, m_pad=cv.cout_pad,
                                k_pad=cv.K_pad, split_k=cv.s_wgrad, split_out=self.kpart_w)
                    C.splitk_reduce(self.kpart_w, cv.s_wgrad, cv.cout_pad * cv.K_pad, master=self._m(cv.entry), lr=lr,
                                    shadow=self._w(cv.entry))
                    self.launches += 1
                else:
                    C.conv_gemm("wgrad", cv.x_in, cv.dz, cv.n, cv.h, cv.w, cv.cin, cv.k, cv.k, cv.pad, m_pad=cv.cout_pad,
                                k_pad=cv.K_pad, sgd_master=self._m(cv.entry), sgd_lr=lr, sgd_shadow=self._w(cv.entry))
                self.launches += 1
                return
            # level 1: the forward ran without a col matrix; build it now, off the forward's critical path
            C.im2col(C.nhwc_view(cv.x_in, cv.n, cv.h, cv.w, cv.cin), cv.col, cv.k, cv.k, cv.stride, cv.pad)
            self.launches += 1
        if self._wgrad_mn:
            # dW[Cout, k] = Σ_pixels dz[pixel, Cout]·col[pixel, k]: both operands are read in place (rows = the
            # reduction index); the Cout padding rows of the tile are TMA zero fill
            if cv.s_wgrad > 1:
                ops.gemm_bf16(cv.dz, cv.col, mn_m=cv.cout_pad, split_k=cv.s_wgrad, split_out=self.kpart_w)
                C.splitk_reduce(self.kpart_w, cv.s_wgrad, cv.cout_pad * cv.K_pad, master=self._m(cv.entry), lr=lr,
                                shadow=self._w(cv.entry))
                self.launches += 1
            else:
                ops.gemm_bf16(cv.dz, cv.col, mn_m=cv.cout_pad, sgd_master=self._m(cv.entry), sgd_lr=lr,
                              sgd_shadow=self._w(cv.entry), sgd_shadow_t=cv.wT if shadow_t else None)
            self.launches += 1
            return
        dzT = self.dzT[: cv.cout_pad * cv.m].view(cv.cout_pad, cv.m)
        if cv.cout_pad != cv.cout:
            dzT[cv.cout:].zero_()
        ops.transpose_bf16(cv.dz, dzT[: cv.cout])
        colT = self.colT[: cv.K_pad * cv.m].view(cv.K_pad, cv.m)
        ops.transpose_bf16(cv.col, colT)
        if cv.s_wgrad > 1:   # partial sums over pixel slices, then one pass: sum + SGD on the master + bf16 shadow
            ops.gemm_bf16(dzT, colT, split_k=cv.s_wgrad, split_out=self.kpart_w)
            C.splitk_reduce(self.kpart_w, cv.s_wgrad, cv.cout_pad * cv.K_pad, master=self._m(cv.entry), lr=lr,
                            shadow=self._w(cv.entry))
            self.launches += 1
        else:
            ops.gemm_bf16(dzT, colT, sgd_master=self._m(cv.entry), sgd_lr=lr, sgd_shadow=self._w(cv.entry),
                          sgd_shadow_t=cv.wT if shadow_t else None)
        self.launches += 3

    def _conv_bwd(self, cv: _Conv, lr: float, dx: Optional[torch.Tensor], add: Optional[torch.Tensor]) -> None:
        """dgrad with the old weights (→ ``dx`` through the col2im gather), then the fused wgrad + SGD.

        With a side stream (``COLEARN_CONV_STREAMS=1``) the wgrad chain (two transposes, GEMM + fused SGD, Wᵀ
        refresh) leaves the critical path: it only needs ``dz`` (event after the BatchNorm backward) and may
        overwrite ``wT`` only once the dgrad GEMM that reads the old weights is done (second event); its scratch
        (``dzT`` / ``colT``) is touched by the side stream alone, ``dcol`` / ``partial`` by the main stream alone."""
        side = self._side
        # Wᵀ straight from the wgrad epilogue (``sgd_shadow_t``) when the layer needs no row padding
        keep_t = self._needs_wT(cv)                      # a W^T copy exists and must follow the update
        in_place = not keep_t                            # the dgrad reads the packed weights the wgrad overwrites
        fuse_t = (self._fuse_shadow_t and cv.cout_pad == cv.cout and cv.s_wgrad == 1 and keep_t
                  and not (cv.implicit and self._implicit >= 2))
        if side is None:
            if dx is not None:
                self._dgrad(cv, dx, add)
            self._wgrad(cv, lr, fuse_t)
            if not fuse_t and keep_t:
                ops.transpose_bf16(self._w(cv.entry)[: cv.cout], cv.wT)
                self.launches += 1
            return
        main = torch.cuda.current_stream(self.dev)
        ev_dz = torch.cuda.Event()
        ev_dz.record(main)
        ev_dgrad = None
        if dx is not None:
            self._dgrad(cv, dx, add)
            ev_dgrad = torch.cuda.Event()
            ev_dgrad.record(main)
        with torch.cuda.stream(side):
            side.wait_event(ev_dz)
            if (fuse_t or in_place) and ev_dgrad is not None:
                side.wait_event(ev_dgrad)                # the epilogue itself overwrites wT (or the W the dgrad reads)
            self._wgrad(cv, lr, fuse_t)
            if not fuse_t and keep_t:
                if ev_dgrad is not None:
                    side.wait_event(ev_dgrad)
                ops.transpose_bf16(self._w(cv.entry)[: cv.cout], cv.wT)
                self.launches += 1

    def backward(self, lr: float) -> None:
        B = self.B
        side = self._side
        if side is not None:
            side.wait_stream(torch.cuda.current_stream(self.dev))    # fork (also what makes it capturable)
        # classifier: dgrad first (old weights), then the fused update
        ops.gemm_bf16(self.dlog, self.fc_wT, out_bf16=self.d_feat)
        ops.transpose_bf16(self.dlog, self.dlogT)
        ops.transpose_bf16(self.feat, self.featT)
        e = self.fc_entry
        ops.gemm_bf16(self.dlogT, self.featT, sgd_master=self._m(e), sgd_lr=lr, sgd_shadow=self._w(e))
        ops.transpose_bf16(self._w(e), self.fc_wT)
        C.avgpool_bwd(self.d_feat, self.d_last, B, self.final_hw, self.feat_dim)
        self.launches += 6
        d_out = self.d_last
        for b in reversed(self.blocks):
            c1, c2, ds = b.c1, b.c2, b.ds
            self._bn_bwd(c2, d_out, True, b.g)                       # through relu(bn2(.) + identity)
            self._conv_bwd(c2, lr, b.d_mid, None)
            self._bn_bwd(c1, b.d_mid, True, None)                    # through relu(bn1(.))
            if ds is None:
                self._conv_bwd(c1, lr, b.d_in, b.g)                  # + identity branch
            else:
                self._bn_bwd(ds, b.g, False, None)
                self._conv_bwd(ds, lr, b.d_skip, None)
                self._conv_bwd(c1, lr, b.d_in, b.d_skip)
            d_out = b.d_in
        st = self.stem
        C.maxpool_bwd(d_out, self.pool_idx, self.d_stem, B, st.oh, st.ow, st.cout, self.pool_k, self.pool_k, self.pool_s, self.pool_p)
        self._bn_bwd(st, self.d_stem, True, None)
        self._conv_bwd(st, lr, None, None)
        if side is not None:
            torch.cuda.current_stream(self.dev).wait_stream(side)    # join: the next forward reads the new shadows
        ops.sgd_step(self.spk, self.gsp, lr)                         # every gamma / beta / fc bias in one launch
        self.launches += 2
        self.steps_done += 1
        self.steps_total += 1

    def step(self, xb: torch.Tensor, labels: torch.Tensor, lr: float) -> torch.Tensor:
        loss = self.forward(xb, labels)
        self.backward(lr)
        return loss

    # -- a whole local fit -------------------------------------------------------------------------------------------------------
    # -- CUDA graph of one SGD step (~320 launches -> one replay) ------------------------------------------------------------
    def _graph_step(self, xb: torch.Tensor, labels: torch.Tensor, lr: float) -> torch.Tensor:
        """Replay the captured step on a new batch.  The first step of a trainer's life runs eagerly (driver entry
        points, allocator pools), the second one is captured; a different lr or input dtype re-captures."""
        key = (float(lr), xb.dtype, tuple(xb.shape))
        if self._graph is None or self._graph_key != key:
            if self.steps_total == 0:
                return self.step(xb, labels, lr)
            self.g_x, self.g_y = torch.zeros_like(xb), torch.zeros_like(labels)
            self.g_loss = torch.zeros((), device=self.dev)
            torch.cuda.synchronize(self.dev)
            graph = torch.cuda.CUDAGraph()
            launches, steps = self.launches, self.steps_done
            with torch.cuda.graph(graph):
                self.g_loss.copy_(self.step(self.g_x, self.g_y, lr))
            self.launches, self.steps_done = launches, steps           # capture executed nothing
            self.steps_total -= 1
            self._graph, self._graph_key = graph, key
        self.g_x.copy_(xb)
        self.g_y.copy_(labels)
        self._graph.replay()
        self.launches += 3
        self.steps_done += 1
        self.steps_total += 1
        return self.g_loss

    def fit(self, flat: torch.Tensor, model: ResNet18, x: torch.Tensor, y: torch.Tensor, cfg, perm: Optional[torch.Tensor],
            use_graph: Optional[bool] = None) -> torch.Tensor:
        """Local SGD in place on ``flat`` (full batches; ``supports`` rejects ragged shards).  On a GPU every step
        after the trainer's first is one CUDA-graph replay."""
        n, B = x.shape[0], self.B
        if use_graph is None:
            use_graph = flat.is_cuda
        step = self._graph_step if use_graph else self.step
        self.load(flat, model)
        labels_all = y.reshape(-1).long()
        limit = cfg.max_nr_batches if cfg.max_nr_batches and cfg.max_nr_batches > 0 else None
        last = torch.zeros((), device=flat.device)
        it = 0
        done = False
        for e in range(cfg.epochs):
            order = perm[e % perm.shape[0]].long() if perm is not None else torch.arange(n, device=flat.device)
            for lo in range(0, n - B + 1, B):
                idx = order[lo:lo + B]
                last = step(x.index_select(0, idx), labels_all.index_select(0, idx), cfg.lr)
                it += 1
                if limit is not None and it >= limit:
                    done = True
                    break
            if done:
                break
        self.store(flat, model)
        return last
