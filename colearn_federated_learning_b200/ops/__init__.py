"""Hot ops.  CUDA tensors → hand-written sm_90a kernels (``csrc/``); CPU tensors → ``reference``.

There is deliberately no silent GPU fallback: a CUDA tensor with the extension missing raises.
"""
from __future__ import annotations

import math
from typing import Optional, Sequence, Tuple

import numpy as np
import torch

from . import reference
from . import _ext
from . import host  # noqa: F401  (native CPU executor of the MLP local fit)
from .fused_mlp import (NET_KINDS, LOSS_CODES, net_kind_for, mlp_local_sgd, mlp_local_sgd_multi, check_class_weights,  # noqa: F401
                        mlp_forward, ClientTask, build_client_descs)
from .reference import make_permutation, total_steps  # noqa: F401


def _cuda(t: torch.Tensor) -> bool:
    return t.is_cuda


def sgd_step(param: torch.Tensor, grad: torch.Tensor, lr: float) -> torch.Tensor:
    """``param -= lr * grad`` in place on a flat fp32 arena (SURVEY K12)."""
    if _cuda(param):
        _ext.require().sgd_step(param, grad.contiguous(), float(lr))
        return param
    return reference.sgd_step(param, grad, lr)


def fedavg_flat(models: torch.Tensor, weights: torch.Tensor) -> torch.Tensor:
    """``sum_k w_k * models[k]``; models ``[K,P]`` fp32, weights ``[K]`` (SURVEY K3)."""
    if _cuda(models):
        return _ext.require().fedavg_flat(models.contiguous(), weights.to(models.device, torch.float32).contiguous())
    return reference.fedavg_flat(models, weights)


# The aggregators a row format refuses, by family, and why (launch_fedavg_apply refuses the same ones)
_REFUSED = {
    "topk": {"coordinate_wise": "top-k sparse deltas: only the (weighted) mean does",
             "distance_based": "top-k sparse deltas: their distances would measure which entries the codec kept, not how far the device "
                               "moved"},
    "secagg": {"coordinate_wise": "secure aggregation: the coordinator only learns the sum",
               "distance_based": "secure aggregation: the masks hide the per-device distances it weighs by"},
}


def _fused_apply(fmt: str, theta: torch.Tensor, k: int, server_lr: float, opt, aggregator, agg_weights_out: Optional[torch.Tensor],
                 launch, reference_apply, distance_rows=None) -> torch.Tensor:
    """What the fused FedAvg applies share, for ``k`` client rows of format ``fmt`` (a key of ``_REFUSED``, or any other name
    for a format that admits every aggregator).  CUDA: ``launch(*tail)`` calls the format's binding with its leading
    arguments followed by the trailing block built here (server step, aggregator, ``agg_weights_out``).  CPU:
    ``agg_weights_out`` of a distance-based aggregator from ``distance_rows() = (rows, weights, start)``, then
    ``reference_apply()``."""
    robust = aggregator is not None and aggregator.robust
    if robust:
        for family, reason in _REFUSED.get(fmt, {}).items():
            if getattr(aggregator, family):
                raise ValueError(f"aggregator {aggregator.kind!r} does not apply to {reason}")
    if opt is not None and float(server_lr) != 1.0:
        raise ValueError(f"server_lr={server_lr} given next to a server optimizer that carries its own lr ({opt.lr})")
    weights_out = agg_weights_out if robust and aggregator.distance_based else None
    if _cuda(theta):
        tail = [float(opt.lr), opt.code, opt.hyper, opt.m, opt.v] if opt is not None else [float(server_lr), 0, [], None, None]
        if robust:
            w = weights_out
            if w is not None and (w.dtype != torch.float32 or not w.is_contiguous() or w.numel() != k or w.device != theta.device):
                raise ValueError(f"agg_weights_out must be a contiguous float32 tensor of {k} elements on {theta.device}")
            tail += [aggregator.code, aggregator.trim, aggregator.iters, aggregator.eps, aggregator.clip, w]
        launch(*tail)
        return theta
    if weights_out is not None:
        rows, weights, start = distance_rows()
        weights_out.copy_(reference.distance_aggregate(rows, weights, aggregator, start)[1])
    return reference_apply()


def fedavg_apply(theta: torch.Tensor, models: torch.Tensor, weights: torch.Tensor, server_lr: float = 1.0, opt=None,
                 aggregator=None, agg_weights_out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """``theta += server_lr * (sum_k w_k models[k] - theta)`` in place (reduce + scale + apply fused).

    ``opt``: a :class:`fl.server_opt.ServerOptState` — the average is followed by that server optimizer's step (FedAvgM /
    FedAdagrad / FedAdam / FedYogi) in the same kernel, with the optimizer's own ``lr``; its moments are updated in place.

    ``aggregator``: a robust :class:`fl.aggregate.Aggregator` (``median`` / ``trimmed_mean``) replaces the weighted sum by
    the coordinate-wise median / trimmed mean of the K models in the same kernel (``weights`` are then not used).  A
    distance-based one (``geomed`` / ``norm_clip``, ``ops/csrc/distance_agg.cuh``) reweights the models by their L2 distance
    from theta (``weights`` are its ``alpha``) in 2 L + 1 launches (``norm_clip``: 3), the last one fused with the step;
    ``agg_weights_out`` (fp32 ``[K]``, optional) then receives every model's final weight, 0 for an excluded one."""
    def launch(*tail):
        _ext.require().fedavg_apply(theta, models.contiguous(), weights.to(theta.device, torch.float32).contiguous(), *tail)

    def reference_apply():
        if opt is None:
            return reference.fedavg_apply(theta, models, weights, server_lr, aggregator=aggregator)
        b1, b2, tau = opt.hyper
        return reference.server_opt_apply(theta, models, weights, opt.kind, opt.lr, opt.m, opt.v, b1, b2, tau, aggregator=aggregator)

    return _fused_apply("fp32", theta, models.shape[0], server_lr, opt, aggregator, agg_weights_out, launch, reference_apply,
                        lambda: (models, weights, theta))


def fedavg_apply_based(theta: torch.Tensor, models: torch.Tensor, ring: torch.Tensor, base_slot, weights: torch.Tensor, write_slot: int,
                       server_lr: float = 1.0, opt=None, aggregator=None, agg_weights_out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """:func:`fedavg_apply` on models trained from older global versions (asynchronous buffered aggregation, ``fl/asyncagg.py``):
    ``ring`` (fp32 ``[slots, P]``, contiguous; ``S + 2`` slots under ``--max-staleness S``) holds the recent versions of
    theta and row ``k`` of ``models [K, >= P]`` counts as its delta ``models[k] - ring[base_slot[k]]``.  ``a = theta + sum_k w_k d_k`` (``fedavg_based_kernel``, fmaf in row
    order), or ``theta +`` the robust aggregate of the deltas (coordinate-wise: unweighted; distance-based: from 0 with
    ``weights`` as alpha), then the server step of ``server_lr`` / ``opt`` as in :func:`fedavg_apply`; the new theta is also
    written to ``ring[write_slot]`` in the same pass.  ``write_slot`` must not be any row's base.  CPU tensors:
    ``reference.fedavg_apply_based``."""
    slots = [int(b) for b in (base_slot.tolist() if isinstance(base_slot, torch.Tensor) else base_slot)]
    if ring.dim() != 2 or ring.shape[1] != theta.numel() or not ring.is_contiguous() or ring.dtype != torch.float32:
        raise ValueError("ring must be a contiguous float32 [slots, P] tensor (it is written in place)")
    if len(slots) != models.shape[0]:
        raise ValueError(f"one base slot per row: {len(slots)} for {models.shape[0]} rows")
    if not 0 <= int(write_slot) < ring.shape[0] or any(not 0 <= b < ring.shape[0] or b == int(write_slot) for b in slots):
        raise ValueError(f"base slots {slots} and write slot {write_slot} must lie in [0, {ring.shape[0]}) and differ")

    def launch(*tail):
        dev = theta.device
        _ext.require().fedavg_apply_based(theta, models.to(dev, torch.float32).contiguous(), ring, torch.tensor(slots, dtype=torch.int32),
                                          weights.to(dev, torch.float32).contiguous(), int(write_slot), *tail)

    return _fused_apply(
        "fp32_based", theta, models.shape[0], server_lr, opt, aggregator, agg_weights_out, launch,
        lambda: reference.fedavg_apply_based(theta, models, ring, slots, weights, write_slot, server_lr, opt=opt, aggregator=aggregator),
        lambda: (reference.based_deltas(models, ring, slots), weights, torch.zeros(theta.numel())))


def _keys_i32(keys, device) -> torch.Tensor:
    """uint32 keys as the int32 tensor (same bits) the kernels take"""
    k = torch.tensor([int(x) & 0xFFFFFFFF for x in keys], dtype=torch.int64)
    return torch.where(k >= 1 << 31, k - (1 << 32), k).to(torch.int32).to(device)


def encode_delta(models: torch.Tensor, theta: torch.Tensor, codec, keys) -> Tuple[torch.Tensor, torch.Tensor]:
    """Quantize the deltas ``models [K, P] - theta [P]`` with the :class:`fl.uplink.UplinkCodec` ``codec`` (int8 / int4)
    and the uint32 rounding ``keys`` (one per row): ``(payload uint8 [K, codec.payload_bytes(P)], scales fp32 [K,
    codec.scale_count(P)])``.  CUDA tensors: ``quantize_delta_kernel`` in one launch (the payload is a view of rows padded
    to 16 bytes); CPU tensors: ``reference.encode_delta``."""
    if not codec.quantized:
        raise ValueError("encode_delta needs an int8 / int4 codec")
    models = models.reshape(len(keys), -1)
    if _cuda(models):
        payload, scales = _ext.require().quantize_delta(models.float().contiguous(), theta.float().contiguous().view(-1),
                                                        _keys_i32(keys, models.device), codec.bits)
        return payload[:, :codec.payload_bytes(theta.numel())], scales
    return reference.encode_delta(models, theta, codec.bits, keys)


def _aligned_rows(payload: torch.Tensor) -> torch.Tensor:
    """the payload with 16-byte aligned rows (the kernels load 8 / 4 bytes per lane): as is when it already has them"""
    if payload.stride(1) == 1 and payload.stride(0) % 16 == 0 and payload.data_ptr() % 16 == 0:
        return payload
    row = (payload.shape[1] + 15) // 16 * 16
    out = torch.zeros(payload.shape[0], row, dtype=torch.uint8, device=payload.device)
    out[:, :payload.shape[1]].copy_(payload)
    return out


def fedavg_apply_quantized(theta: torch.Tensor, payload: torch.Tensor, scales: torch.Tensor, weights: torch.Tensor, codec,
                           server_lr: float = 1.0, opt=None, aggregator=None, agg_weights_out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """:func:`fedavg_apply` on quantized deltas (``encode_delta``'s output, or the same bytes from the wire): ``a = theta +
    sum_k w_k d^_k`` (or ``theta +`` the robust aggregate of the decoded deltas) and the server step towards ``a``, decode
    fused into the reduce (``fedavg_q_kernel`` / ``fedavg_q_robust_kernel``).  ``opt`` / ``aggregator`` as in
    :func:`fedavg_apply`; a distance-based ``aggregator`` measures the decoded deltas from 0 (``fedavg_q`` loaders decode
    inside every pass), ``agg_weights_out`` as in :func:`fedavg_apply`.  CPU tensors: ``reference.fedavg_apply_quantized``."""
    if not codec.quantized:
        raise ValueError("fedavg_apply_quantized needs an int8 / int4 codec")
    k = payload.shape[0]

    def launch(*tail):
        dev = theta.device
        w = weights if weights is not None else torch.full((k,), 1.0 / k)   # (a coordinate-wise aggregator does not read them)
        _ext.require().fedavg_apply_quantized(theta, _aligned_rows(payload.to(dev)), scales.to(dev, torch.float32).contiguous(),
                                              w.to(dev, torch.float32).contiguous(), codec.bits, *tail)

    return _fused_apply(
        codec.kind, theta, k, server_lr, opt, aggregator, agg_weights_out, launch,
        lambda: reference.fedavg_apply_quantized(theta, payload, scales, weights, codec.bits, server_lr, opt=opt, aggregator=aggregator),
        lambda: (reference.decode_delta(payload, scales, codec.bits, theta.numel()), weights, torch.zeros(theta.numel())))


def encode_topk_delta(models: torch.Tensor, theta: torch.Tensor, residual: torch.Tensor, codec) -> Tuple[torch.Tensor, torch.Tensor]:
    """Top-``codec.k`` sparsification with error feedback of ``v = (models [K, P] - theta [P]) + residual [K, P]``:
    ``(indices uint8 [K, E], values fp32 [K, E])`` with ``E = codec.entries(P)``, and ``residual`` (fp32, contiguous)
    overwritten in place with what was not sent.  CUDA tensors: ``topk_delta_kernel`` in one launch; CPU tensors:
    ``reference.encode_topk_delta``."""
    if not codec.sparse:
        raise ValueError("encode_topk_delta needs a topk codec")
    if residual.dtype != torch.float32 or not residual.is_contiguous() or residual.dim() != 2:
        raise ValueError("residual must be a contiguous float32 [K, P] tensor (it is updated in place)")
    models = models.reshape(residual.shape)
    if _cuda(models):
        idx, val = _ext.require().topk_delta(models.float().contiguous(), theta.float().contiguous().view(-1), residual, codec.k)
        return idx, val
    return reference.encode_topk_delta(models, theta, residual, codec.k)


def fedavg_apply_topk(theta: torch.Tensor, indices: torch.Tensor, values: torch.Tensor, weights: torch.Tensor, codec,
                      server_lr: float = 1.0, opt=None, aggregator=None) -> torch.Tensor:
    """:func:`fedavg_apply` on top-k sparse deltas (``encode_topk_delta``'s output, or the same bytes from the wire): ``a =
    theta + sum_k w_k d_k`` and the server step towards ``a`` (``server_lr``, or the server optimizer ``opt`` as in
    :func:`fedavg_apply`), decode fused into the reduce (``fedavg_topk_kernel``).  A robust ``aggregator`` is refused: a
    coordinate-wise median of k/256-sparse deltas is 0 wherever fewer than half the devices sent that coordinate, so it
    would throw the update away.  CPU tensors: ``reference.fedavg_apply_topk``."""
    if not codec.sparse:
        raise ValueError("fedavg_apply_topk needs a topk codec")

    def launch(*tail):
        dev = theta.device
        _ext.require().fedavg_apply_topk(theta, indices.to(dev, torch.uint8).contiguous(), values.to(dev, torch.float32).contiguous(),
                                         weights.to(dev, torch.float32).contiguous(), codec.k, *tail)

    return _fused_apply("topk", theta, indices.shape[0], server_lr, opt, aggregator, None, launch,
                        lambda: reference.fedavg_apply_topk(theta, indices, values, weights, codec.k, server_lr, opt=opt))


def encode_downlink(theta: torch.Tensor, replica: torch.Tensor, codec, key: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """The coordinator's downlink (``ops/csrc/downlink.cuh``): the wire of ``theta [P] - replica [P]`` with the
    :class:`fl.uplink.UplinkCodec` ``codec``, and ``replica`` (contiguous fp32) advanced in place by what it carries.  int8 /
    int4: ``(payload uint8 [codec.payload_bytes(P)], scales fp32 [codec.scale_count(P)])`` rounded with the uint32 ``key``;
    topk: ``(indices uint8 [E], values fp32 [E])``.  CUDA tensors: ``downlink_quant_kernel`` / ``downlink_topk_kernel`` in one
    launch; CPU tensors: ``reference.encode_downlink``."""
    if not (codec.quantized or codec.sparse):
        raise ValueError("encode_downlink needs an int8 / int4 / topk codec")
    if replica.dtype != torch.float32 or not replica.is_contiguous() or replica.numel() != theta.numel():
        raise ValueError("the replica must be a contiguous float32 tensor of theta's size (it is updated in place)")
    if _cuda(replica):
        th = theta.to(replica.device, torch.float32).contiguous().view(-1)
        if codec.quantized:
            payload, scales = _ext.require().downlink_quant(th, replica.view(-1), int(key) & 0xFFFFFFFF, codec.bits)
            return payload[:codec.payload_bytes(theta.numel())], scales
        return tuple(_ext.require().downlink_topk(th, replica.view(-1), codec.k))
    return reference.encode_downlink(theta, replica, codec, key)


def apply_downlink(replica: torch.Tensor, a: torch.Tensor, b: torch.Tensor, codec) -> torch.Tensor:
    """A device's side of the downlink: ``replica`` (contiguous fp32) advanced in place by a wire ``(a, b)`` that passed the
    reply checks (``(payload, scales)`` for int8 / int4, ``(indices, values)`` for topk).  CUDA tensors:
    ``replica_apply_q_kernel`` / ``replica_apply_topk_kernel``; CPU tensors: ``reference.apply_downlink``."""
    if not (codec.quantized or codec.sparse):
        raise ValueError("apply_downlink needs an int8 / int4 / topk codec")
    if replica.dtype != torch.float32 or not replica.is_contiguous():
        raise ValueError("the replica must be a contiguous float32 tensor (it is updated in place)")
    if _cuda(replica):
        dev = replica.device
        if codec.quantized:
            payload = _aligned_rows(a.to(dev, torch.uint8).reshape(1, -1)).reshape(-1)
            _ext.require().replica_apply_quant(replica.view(-1), payload, b.to(dev, torch.float32).contiguous(), codec.bits)
        else:
            _ext.require().replica_apply_topk(replica.view(-1), a.to(dev, torch.uint8).contiguous(), b.to(dev, torch.float32).contiguous(),
                                              codec.k)
        return replica
    return reference.apply_downlink(replica, a, b, codec)


def secagg_key_words(keys, device=None) -> torch.Tensor:
    """int32 ``[S, 8]`` (the little-endian words, as the kernels take them) of ``S`` 32-byte stream keys"""
    return torch.from_numpy(reference._key_words(keys).view(np.int32).copy()).to(device)


def _secagg_streams_args(keys, signs, device):
    kw = keys.to(device, torch.int32).contiguous() if isinstance(keys, torch.Tensor) else secagg_key_words(keys, device)
    sg = torch.as_tensor(signs.cpu() if isinstance(signs, torch.Tensor) else list(signs), dtype=torch.int32).reshape(-1)
    if sg.numel() != kw.shape[0] or not bool(((sg == 1) | (sg == -1)).all()):
        raise ValueError("one sign (+1 / -1) per stream key")
    return kw, sg.to(device)


def secagg_mask(model: torch.Tensor, theta: torch.Tensor, keys, signs, clip: float, frac_bits: int) -> Tuple[torch.Tensor, int, int]:
    """A device's masked update for secure aggregation (``ops/csrc/secagg.cuh``, ``fl/secagg.py``): ``(y uint32 [P], clipped,
    nonfinite)`` with ``y = enc(model - theta) + sum_s signs[s] PRG(keys[s])`` (mod 2^32), ``enc`` the fixed-point code with
    clip ``clip`` and ``frac_bits`` fraction bits, ``keys`` 32-byte ChaCha20 keys (or their ``[S, 8]`` int32 words) and
    ``signs`` +1 / -1.  CUDA tensors: ``secagg_mask_kernel`` in one launch; CPU tensors: ``reference.secagg_mask``."""
    if not (math.isfinite(clip) and clip > 0):
        raise ValueError(f"the clip must be finite and > 0, not {clip}")
    if _cuda(theta):
        kw, sg = _secagg_streams_args(keys, signs, theta.device)
        out, counts = _ext.require().secagg_mask(model.to(theta.device, torch.float32).contiguous().view(-1),
                                                 theta.float().contiguous().view(-1), kw, sg, float(clip), int(frac_bits))
        c = counts.tolist()
        return out.view(torch.uint32), int(c[0]), int(c[1])
    return reference.secagg_mask(model, theta, keys, signs, clip, frac_bits)


def fedavg_apply_secagg(theta: torch.Tensor, masked: torch.Tensor, keys, signs, frac_bits: int, n: int, server_lr: float = 1.0,
                        opt=None, aggregator=None) -> torch.Tensor:
    """Secure aggregation's unmask + decode + FedAvg apply in place: ``z = sum_k masked[k] + sum_s signs[s] PRG(keys[s])``
    (mod 2^32; the correction streams are the survivors' self masks and the pair masks of the dropped devices, negated),
    ``mean = (float)(int32)z 2^-frac_bits / n``, ``a = theta + mean``, then ``theta += server_lr (a - theta)`` or the server
    optimizer step of ``opt`` (as in :func:`fedavg_apply`).  ``masked``: uint32 (or int32 with the same bits) ``[K, P]``.  A
    robust ``aggregator`` is refused: only a sum survives the masks.  CUDA tensors: ``fedavg_secagg_kernel`` (after
    ``secagg_streams_kernel`` when the streams are split); CPU tensors: ``reference.fedavg_apply_secagg``."""
    if int(n) < 1:
        raise ValueError("the mean needs n >= 1 survivors")

    def launch(*tail):
        dev = theta.device
        kw, sg = _secagg_streams_args(keys, signs, dev)
        rows = masked.to(dev).contiguous().view(torch.int32).reshape(-1, theta.numel())
        _ext.require().fedavg_apply_secagg(theta, rows, kw, sg, int(frac_bits), int(n), *tail)

    return _fused_apply("secagg", theta, masked.shape[0], server_lr, opt, aggregator, None, launch,
                        lambda: reference.fedavg_apply_secagg(theta, masked, keys, signs, frac_bits, n, server_lr, opt=opt))


def sigmoid_bce(z: torch.Tensor, y: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """(mean BCE(sigmoid(z), y), dL/dz) in one pass (SURVEY K9)."""
    if _cuda(z):
        loss, dz = _ext.require().sigmoid_bce(z.contiguous().float(), y.contiguous().float().view_as(z))
        return loss, dz
    return reference.sigmoid_bce(z, y)


def sse_loss(out: torch.Tensor, y: torch.Tensor, mean: bool = False) -> Tuple[torch.Tensor, torch.Tensor]:
    """(sum (out-y)^2 [/batch], gradient) (SURVEY K11)."""
    if _cuda(out):
        scale = 1.0 / out.shape[0] if mean else 1.0
        loss, dz = _ext.require().sse_loss(out.contiguous().float(), y.contiguous().float().view_as(out), scale)
        return loss, dz
    return reference.loss_and_dz(out, y, "mse" if mean else "sse", "none")


def softmax_xent(logits: torch.Tensor, labels: torch.Tensor, bf16_grad: bool = False) -> Tuple[torch.Tensor, torch.Tensor]:
    """(mean softmax cross-entropy, dL/dlogits) in one pass (SURVEY K10).

    The kernel does not check ``labels``: a row whose label is outside ``[0, cols)`` adds nothing to the loss and gets
    the plain softmax as its gradient, with no error.  The CPU path raises on it."""
    if _cuda(logits):
        loss, dl = _ext.require().softmax_xent(logits.contiguous(), labels.contiguous().long().view(-1), bool(bf16_grad))
        return loss, dl
    loss, dl = reference.softmax_xent(logits, labels)
    return loss, (dl.to(torch.bfloat16) if bf16_grad else dl)


def eval_binary(p: torch.Tensor, y: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """(sum BCE, #correct round(p)==y) (SURVEY K15; reference ``evaluate`` cf.py:233-253)."""
    if _cuda(p):
        loss, correct = _ext.require().eval_binary(p.contiguous().float().view(-1), y.contiguous().float().view(-1))
        return loss, correct
    return reference.eval_binary(p, y)


def eval_summary(scores: torch.Tensor, labels: torch.Tensor, bins: int = 256, threshold: float = 0.5,
                 segments: Optional[Sequence[int]] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """Detection-metrics summary of model outputs (``ops/csrc/eval_summary.cuh``): ``(counts int64 [S, L], loss_sum float64
    [S])``, one row per segment of consecutive rows.  ``scores``: ``[N, C]`` (or ``[N]``) fp32 outputs after the output
    activation, ``labels``: ``[N]``, ``segments``: the row count of every segment (one segment of all rows when None).  Row
    ``s`` of ``counts`` holds ``n``, ``n_invalid``, the ``C' x C'`` confusion matrix and the ``C x 2 x bins`` score histograms
    (``fl/fedeval.py`` reads them).  CUDA tensors: one memset and one ``eval_summary_kernel`` launch; CPU tensors:
    ``reference.eval_summary``."""
    scores = scores.view(-1, 1) if scores.dim() == 1 else scores
    n = scores.shape[0]
    sizes = [n] if segments is None else [int(s) for s in segments]
    if any(s < 0 for s in sizes) or sum(sizes) != n or not sizes:
        raise ValueError(f"segments {sizes} do not cover the {n} rows")
    offsets = [0]
    for s in sizes:
        offsets.append(offsets[-1] + s)
    reference.eval_summary_limits(scores.shape[1], int(bins), float(threshold), n)
    if _cuda(scores):
        counts, loss = _ext.require().eval_summary(scores.float().contiguous(), labels.to(scores.device, torch.float32).contiguous().view(-1),
                                                   torch.tensor(offsets, dtype=torch.int64), int(bins), float(threshold), 0)
        return counts, loss
    return reference.eval_summary(scores, labels, int(bins), float(threshold), offsets)


def recon_summary(xhat: torch.Tensor, x: torch.Tensor, labels: Optional[torch.Tensor] = None, bins: int = 256,
                  segments: Optional[Sequence[int]] = None, alarm_bin: Optional[int] = None):
    """Reconstruction-error summary of an autoencoder's outputs (``ops/csrc/recon_summary.cuh``): ``(counts int64 [S, 2 + 2 B],
    err_sum float64 [S], err fp32 [N] or None, flag uint8 [N] or None)``, one row per segment of consecutive rows.  ``xhat``:
    the model's output ``[N, D]``, ``x``: its input, ``labels``: ``[N]`` 0 / 1 or None, ``segments``: the row count of every
    segment (one segment of all rows when None).  Row ``s`` of ``counts`` holds ``n``, ``n_invalid`` and the error
    histograms of label 0 and label 1 (``fl/anomaly.py`` reads them).  With ``alarm_bin`` also the per-row error and alarm
    flag.  CUDA tensors: one memset and one ``recon_summary_kernel`` launch; CPU tensors: ``reference.recon_summary``."""
    n = x.shape[0]
    sizes = [n] if segments is None else [int(s) for s in segments]
    if any(s < 0 for s in sizes) or sum(sizes) != n or not sizes:
        raise ValueError(f"segments {sizes} do not cover the {n} rows")
    offsets = [0]
    for s in sizes:
        offsets.append(offsets[-1] + s)
    if xhat.dim() != 2 or tuple(xhat.shape) != tuple(x.shape):
        raise ValueError(f"xhat {tuple(xhat.shape)} and x {tuple(x.shape)} must both be [N, D]")
    reference.recon_summary_limits(int(x.shape[1]), int(bins), n, alarm_bin)
    if _cuda(x):
        lab = None if labels is None else labels.to(x.device, torch.float32).contiguous().view(-1)
        counts, total, err, flag = _ext.require().recon_summary(xhat.to(x.device).float().contiguous(), x.float().contiguous(), lab,
                                                                torch.tensor(offsets, dtype=torch.int64), int(bins),
                                                                -1 if alarm_bin is None else int(alarm_bin), 0)
        return counts, total, (err if alarm_bin is not None else None), (flag if alarm_bin is not None else None)
    return reference.recon_summary(xhat, x, labels, int(bins), offsets, alarm_bin)


def argmax_rows(x: torch.Tensor) -> torch.Tensor:
    """``x.argmax(1, keepdim=True)`` (SURVEY K16; reference inference fc.py:252-256)."""
    if _cuda(x):
        return _ext.require().argmax_rows(x.contiguous().float())
    return reference.argmax_rows(x)


def minmax_scale(x: torch.Tensor) -> torch.Tensor:
    """Column-wise scale to [0,1] (SURVEY K13; reference ``MinMaxScaler`` ds.py:31-32): ``(x - lo) / (hi - lo)``, a
    constant column to 0.  NaN entries are left out of a column's min and max, as sklearn's ``MinMaxScaler`` does, and
    scale to NaN; on both paths.  ``minmax_scale_kernel`` multiplies by ``1 / (hi - lo)`` where this path divides: the
    two may differ in the last bit (the kernel's maximum can be 1 - 2^-24)."""
    if _cuda(x):
        return _ext.require().minmax_scale(x.contiguous().float())
    nan = torch.isnan(x)
    lo = torch.where(nan, torch.inf, x).amin(0)
    rng = torch.where(nan, -torch.inf, x).amax(0) - lo
    rng = torch.where(rng == 0, torch.ones_like(rng), rng)
    return (x - lo) / rng


def device_permutation(n: int, rows: int, seed: int, device) -> torch.Tensor:
    """int32 ``[rows, n]`` keyed random permutations generated on the device (SURVEY K14).  A
    4-round Feistel bijection with cycle walking: every index is computed independently, so no
    H2D traffic and no serial Fisher-Yates.  CPU: ``reference.make_permutation``."""
    device = torch.device(device)
    if device.type == "cuda":
        return _ext.require().feistel_permutation(int(n), int(rows), int(seed), device)
    return reference.make_permutation(n, rows, seed)


def fp32_to_bf16(x: torch.Tensor) -> torch.Tensor:
    if _cuda(x):
        return _ext.require().fp32_to_bf16(x.contiguous())
    return x.to(torch.bfloat16)


def l2_flush(buf: torch.Tensor) -> None:
    """Overwrite a >L2-sized buffer (bench hygiene between timed iterations)."""
    if _cuda(buf):
        _ext.require().l2_flush(buf)
    else:
        buf.fill_(1.0)


from .linear import gemm_bf16, linear_forward, transpose_bf16, bias_sgd_from_partials, local_opt_apply  # noqa: E402,F401
