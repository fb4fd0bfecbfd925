"""Plain-PyTorch fp32 definitions of every op in ``ops/`` .

Two jobs: (1) the numerics oracle each sm_90a kernel is tested against, (2) the CPU execution
path (BASELINE config 1 runs with no GPU; multi-process CPU tests run over gloo).  Nothing here
is on the GPU hot path — on a CUDA box the dispatchers in ``ops/__init__`` refuse to fall back
to these silently.

The local-SGD semantics re-create PySyft's ``FederatedClient._fit`` (SURVEY C27, [EXTERNAL]):
``for epoch: for batch in shuffled(data): zero_grad; out = model(x); loss = loss_fn(out, y);
backward; SGD step; if ++it >= max_nr_batches >= 0: stop`` and return the last loss.
"""
from __future__ import annotations

import math
from typing import List, Optional, Sequence, Tuple

import numpy as np
import torch

LOSSES = ("bce", "sse", "xent", "mse")


# ------------------------------------------------------------------------------------------------
# flat-arena helpers
# ------------------------------------------------------------------------------------------------
def mlp_views(flat: torch.Tensor, dims: Sequence[int]) -> List[Tuple[torch.Tensor, torch.Tensor]]:
    """[(W[out,in], b[out])] views into the flat arena (state-dict order)."""
    out, off = [], 0
    for i in range(len(dims) - 1):
        k, n = dims[i], dims[i + 1]
        w = flat[off:off + k * n].view(n, k)
        off += k * n
        b = flat[off:off + n]
        off += n
        out.append((w, b))
    return out


def mlp_forward(flat: torch.Tensor, dims: Sequence[int], x: torch.Tensor,
                out_activation: str = "none") -> Tuple[torch.Tensor, List[torch.Tensor]]:
    """Returns (output, [input of every layer]) — activations are kept for the backward."""
    acts = []
    h = x
    views = mlp_views(flat, dims)
    for li, (w, b) in enumerate(views):
        acts.append(h)
        h = h @ w.t() + b
        if li < len(views) - 1:
            h = torch.relu(h)
    if out_activation == "sigmoid":
        h = torch.sigmoid(h)
    return h, acts


def loss_and_dz(out: torch.Tensor, y: torch.Tensor, loss: str, out_activation: str
                ) -> Tuple[torch.Tensor, torch.Tensor]:
    """Loss value and gradient w.r.t. the last layer's *pre-activation*.

    bce  : mean binary cross-entropy on probabilities (reference remote mode, cf.py:76-79).
           Needs a sigmoid head; log terms are clamped at -100 like ``F.binary_cross_entropy``.
    sse  : sum of squared errors (reference local mode, cf.py:112).
    mse  : sse / batch (reference encrypted mode, cf.py:158).
    xent : softmax cross-entropy, integer labels in ``y[:, 0]``, mean over the batch.
    """
    bsz = out.shape[0]
    if loss == "xent":
        labels = y.reshape(bsz).long()
        lse = torch.logsumexp(out, dim=1)
        value = (lse - out.gather(1, labels.view(-1, 1)).squeeze(1)).mean()
        p = torch.softmax(out, dim=1)
        p = p - torch.nn.functional.one_hot(labels, out.shape[1]).to(p.dtype)
        return value, p / bsz
    y = y.reshape(out.shape).to(out.dtype)
    if loss == "bce":
        if out_activation != "sigmoid":
            raise ValueError("bce needs a sigmoid head")
        logp = torch.clamp(torch.log(out), min=-100.0)
        log1mp = torch.clamp(torch.log1p(-out), min=-100.0)
        value = -(y * logp + (1 - y) * log1mp).mean()
        return value, (out - y) / out.numel()
    if loss in ("sse", "mse"):
        diff = out - y
        scale = 1.0 if loss == "sse" else 1.0 / bsz
        value = (diff * diff).sum() * scale
        dz = 2.0 * diff * scale
        if out_activation == "sigmoid":
            dz = dz * out * (1 - out)
        return value, dz
    raise ValueError(f"unknown loss {loss!r}")


def mlp_backward(flat: torch.Tensor, dims: Sequence[int], acts: List[torch.Tensor],
                 dz: torch.Tensor) -> torch.Tensor:
    """Gradient of the flat arena given d(loss)/d(pre-activation of the last layer)."""
    grad = torch.zeros_like(flat)
    gviews = mlp_views(grad, dims)
    views = mlp_views(flat, dims)
    for li in range(len(views) - 1, -1, -1):
        w, _ = views[li]
        gw, gb = gviews[li]
        a = acts[li]
        gw.copy_(dz.t() @ a)
        gb.copy_(dz.sum(0))
        if li > 0:
            # a = relu(z_{li-1}); ReLU's backward as autograd computes it: 0 where a <= 0, so a NaN activation passes dz on
            dz = torch.ops.aten.threshold_backward(dz @ w, a, 0)
    return grad


def mlp_grad(flat, dims, x, y, loss="xent", out_activation="none"):
    out, acts = mlp_forward(flat, dims, x, out_activation)
    value, dz = loss_and_dz(out, y, loss, out_activation)
    return value, mlp_backward(flat, dims, acts, dz)


# ------------------------------------------------------------------------------------------------
# local SGD (the worker-side fit loop)
# ------------------------------------------------------------------------------------------------
def make_permutation(n: int, epochs: int, seed: int, device=None, shuffle: bool = True) -> torch.Tensor:
    """int32 ``[epochs, n]`` sample order.  CPU generator => identical on every backend."""
    g = torch.Generator().manual_seed(int(seed))
    rows = [torch.randperm(n, generator=g) if shuffle else torch.arange(n) for _ in range(epochs)]
    perm = torch.stack(rows).to(torch.int32)
    return perm.to(device) if device is not None else perm


def total_steps(n: int, batch_size: int, epochs: int, max_nr_batches: int = -1) -> int:
    """Number of SGD steps a fit performs (``max_nr_batches <= 0`` means unlimited)."""
    steps = epochs * math.ceil(n / batch_size)
    if max_nr_batches is not None and max_nr_batches > 0:
        steps = min(steps, max_nr_batches)
    return steps


def mlp_local_sgd(flat: torch.Tensor, dims: Sequence[int], x: torch.Tensor, y: torch.Tensor,
                  perm: torch.Tensor, batch_size: int = 1, lr: float = 0.01, epochs: int = 1,
                  max_nr_batches: int = -1, loss: str = "xent", out_activation: str = "none"
                  ) -> torch.Tensor:
    """In-place local SGD on the flat arena; returns the last batch's loss (0-dim tensor).

    ``max_nr_batches``: PySyft stops when ``it >= max_nr_batches >= 0`` *after* a step, so 0
    behaves like "one step"; negative means unlimited.  We normalise: <= 0 → unlimited except
    that the reference never passes 0 (default -1, round mode 1000)."""
    n = x.shape[0]
    it = 0
    last = torch.zeros((), dtype=flat.dtype, device=flat.device)
    limit = max_nr_batches if (max_nr_batches is not None and max_nr_batches > 0) else None
    for e in range(epochs):
        order = perm[e % perm.shape[0]].long()
        for lo in range(0, n, batch_size):
            idx = order[lo:lo + batch_size]
            last, g = mlp_grad(flat, dims, x[idx], y[idx], loss, out_activation)
            flat.sub_(lr * g)
            it += 1
            if limit is not None and it >= limit:
                return last
    return last


# ------------------------------------------------------------------------------------------------
# standalone fused-op references
# ------------------------------------------------------------------------------------------------
def sigmoid_bce(z: torch.Tensor, y: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """(mean BCE of sigmoid(z), d/dz)."""
    p = torch.sigmoid(z)
    return loss_and_dz(p, y, "bce", "sigmoid")


def softmax_xent(logits: torch.Tensor, labels: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    return loss_and_dz(logits.float(), labels.view(-1, 1), "xent", "none")


def sse_loss(out: torch.Tensor, y: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    return loss_and_dz(out, y, "sse", "none")


def sgd_step(param: torch.Tensor, grad: torch.Tensor, lr: float) -> torch.Tensor:
    return param.sub_(grad.to(param.dtype), alpha=lr)


def fedavg_flat(models: torch.Tensor, weights: torch.Tensor) -> torch.Tensor:
    """``sum_k w_k * models[k]``; models ``[K, P]``, weights ``[K]`` (already normalised)."""
    return (weights.view(-1, 1).to(models.dtype) * models).sum(0)


def agg_trim_count(kind: str, beta: float, n: int) -> int:
    """Values dropped at each end of ``n`` sorted ones (``fl/aggregate.py``); ``beta * n`` is formed in float32."""
    half = (n - 1) // 2
    if kind == "median":
        return half
    if kind == "trimmed_mean":
        return min(int(math.floor(np.float32(beta) * np.float32(n))), half)
    raise ValueError(f"not a robust aggregator: {kind!r}")


def robust_aggregate(models: torch.Tensor, mask: Optional[int] = None, kind: str = "median", beta: float = 0.0) -> torch.Tensor:
    """Coordinate-wise median / trimmed mean of the rows ``k`` of ``models [K, P]`` set in the bitmask ``mask`` (all rows if
    None), the definition the kernels (``ops/csrc/robust_agg.cuh``) match bit for bit: int32 keys of the IEEE total order, rank
    = #smaller keys + #equal keys in earlier rows, a sequential float32 sum of the kept rows in row order, one division.
    Returns ``[P]``; no row selected is an error (the caller keeps theta)."""
    rows = [k for k in range(models.shape[0]) if mask is None or (mask >> k) & 1]
    n = len(rows)
    if n == 0:
        raise ValueError("robust_aggregate: no model contributes")
    v = models[rows].float().contiguous()
    bits = v.view(torch.int32)
    key = bits ^ ((bits >> 31) & 0x7FFFFFFF)
    b = agg_trim_count(kind, beta, n)
    acc = torch.zeros(v.shape[1], dtype=torch.float32, device=v.device)
    for k in range(n):
        rank = (key < key[k]).sum(0) + (key[:k] == key[k]).sum(0)
        acc = acc + torch.where((rank >= b) & (rank < n - b), v[k], torch.zeros_like(v[k]))
    return acc / torch.full_like(acc, float(n - 2 * b))


DA_CHUNK = 2048      # elements per chunk of the distance sums (ops/csrc/distance_agg.cuh: one CTA x 8 elements per lane)
DA_THREADS = 256


def _da_tree(v: torch.Tensor) -> torch.Tensor:
    """float64 ``[..., 256]`` lane values -> ``[...]``: the halving tree over the 32 lanes of each warp, then the 8 warp
    sums in warp order (the in-CTA order of ``distance_agg.cuh``)."""
    a = v.reshape(*v.shape[:-1], DA_THREADS // 32, 32).clone()
    o = 16
    while o:
        a[..., :o] = a[..., :o] + a[..., o:2 * o]
        o >>= 1
    t = a[..., 0, 0]
    for w in range(1, DA_THREADS // 32):
        t = t + a[..., w, 0]
    return t


def distance_sq(rows: torch.Tensor, c: torch.Tensor) -> torch.Tensor:
    """float64 ``[K]``: ``sum_j (rows[k, j] - c[j])^2`` in the order of ``distance_agg.cuh`` (float32 difference, float64
    squares; a lane's 8 elements in order, the in-CTA tree per 2048-element chunk, the chunks strided over 256 lanes in
    ascending order, the same tree).  Bit for bit what the kernels compute."""
    K, P = rows.shape
    nch = (P + DA_CHUNK - 1) // DA_CHUNK
    d = torch.zeros(K, nch * DA_CHUNK, dtype=torch.float32)
    d[:, :P] = rows.float().cpu() - c.float().cpu().view(1, -1)
    d = d.double().reshape(K, nch, DA_THREADS, 8)
    lane = torch.zeros(K, nch, DA_THREADS, dtype=torch.float64)
    for i in range(8):
        lane = lane + d[..., i] * d[..., i]          # the square of a float32 is exact in float64: = fma(d, d, lane)
    part = _da_tree(lane)                              # [K, nch]
    m = (nch + DA_THREADS - 1) // DA_THREADS
    pad = torch.zeros(K, m * DA_THREADS, dtype=torch.float64)
    pad[:, :nch] = part
    pad = pad.reshape(K, m, DA_THREADS)
    acc = torch.zeros(K, DA_THREADS, dtype=torch.float64)
    for i in range(m):
        acc = acc + pad[:, i]
    return _da_tree(acc)


def distance_weights(aggregator, alpha: torch.Tensor, d: torch.Tensor) -> Tuple[torch.Tensor, bool]:
    """(float32 ``[K]`` weights, any row left) from the distances ``d`` (float64) and the FedAvg weights ``alpha``:
    ``distance_agg.cuh``'s da_raw / da_weight, the raw weights summed in row order."""
    a = alpha.detach().float().cpu().double().tolist()
    dl = d.tolist()
    kept = [math.isfinite(x) for x in dl]
    geo = aggregator.kind == "geomed"
    eps = float(np.float32(aggregator.eps))
    tau = float(np.float32(aggregator.clip))
    raw = [(a[k] / max(eps, dl[k]) if geo else a[k]) if kept[k] else 0.0 for k in range(len(dl))]
    tot = 0.0
    for r in raw:
        tot += r
    live = sum(kept) > 0 and tot > 0.0
    w = [0.0] * len(dl)
    if live:
        for k in range(len(dl)):
            if kept[k]:
                w[k] = raw[k] / tot if geo else raw[k] / tot * min(1.0, tau / dl[k] if dl[k] > 0 else math.inf)
    return torch.tensor(w, dtype=torch.float64).float(), live


def _fmaf_rows(w: torch.Tensor, rows: torch.Tensor) -> torch.Tensor:
    """``sum_k fmaf(w_k, rows[k], acc)`` in row order from +0, rows of weight 0 skipped (float32 multiply and add: within an
    ulp per step of the kernels' fmaf)."""
    acc = torch.zeros(rows.shape[1], dtype=torch.float32)
    for k in range(rows.shape[0]):
        if float(w[k]) != 0.0:
            acc = acc + w[k] * rows[k]
    return acc


def distance_aggregate(rows: torch.Tensor, alpha: torch.Tensor, aggregator, start: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """The distance-based aggregate of ``ops/csrc/distance_agg.cuh`` (``geomed`` / ``norm_clip``) of ``rows [K, P]`` from
    the start point ``start [P]`` (theta for models, 0 for deltas) with the FedAvg weights ``alpha [K]``: ``(a [P], final
    weights float32 [K])``, weight 0 for an excluded row.  With no row left, ``a`` is the start point."""
    x = rows.detach().float().cpu()
    c0 = start.detach().float().cpu().reshape(-1)
    w, live = distance_weights(aggregator, alpha, distance_sq(x, c0).sqrt())
    if aggregator.kind == "norm_clip":
        acc = torch.zeros_like(c0)
        for k in range(x.shape[0]):
            if float(w[k]) != 0.0:
                acc = acc + w[k] * (x[k] - c0)
        return c0 + acc, w
    for _ in range(aggregator.iters - 1):
        c = _fmaf_rows(w, x) if live else c0
        w, live = distance_weights(aggregator, alpha, distance_sq(x, c).sqrt())
    return (_fmaf_rows(w, x) if live else c0.clone()), w


def aggregate(models: torch.Tensor, weights: torch.Tensor, aggregator=None, start: Optional[torch.Tensor] = None) -> torch.Tensor:
    """The average the server steps towards: :func:`fedavg_flat` (``aggregator`` None or ``mean``),
    :func:`robust_aggregate` over all rows (unweighted) or :func:`distance_aggregate` from ``start``."""
    if aggregator is None or not aggregator.robust:
        return fedavg_flat(models, weights)
    if aggregator.distance_based:
        a, _ = distance_aggregate(models, weights, aggregator, start)
        return a.to(models.device)
    return robust_aggregate(models, None, aggregator.kind, aggregator.trim)


def fedavg_apply(theta: torch.Tensor, models: torch.Tensor, weights: torch.Tensor,
                 server_lr: float = 1.0, aggregator=None) -> torch.Tensor:
    """``theta <- theta + server_lr * (sum_k w_k models[k] - theta)`` (weights sum to 1).  ``aggregator``: a robust
    :class:`fl.aggregate.Aggregator` replaces the weighted sum by its unweighted aggregate."""
    avg = aggregate(models, weights, aggregator, theta)
    return theta.add_(server_lr * (avg - theta))


def server_opt_step(theta: torch.Tensor, avg: torch.Tensor, kind: str, lr: float, m=None, v=None, beta1: float = 0.9,
                    beta2: float = 0.99, tau: float = 1e-3) -> torch.Tensor:
    """One server optimizer step towards the FedAvg average ``avg`` (``fl/server_opt.py`` has the table), in place on
    ``theta`` and the moments ``m`` / ``v``.  ``sgd`` is exactly :func:`fedavg_apply`'s update."""
    d = avg - theta
    if kind == "sgd":
        return theta.add_(lr * d)
    if kind == "avgm":
        m.mul_(beta1).add_(d)
        return theta.add_(lr * m)
    m.mul_(beta1).add_((1.0 - beta1) * d)
    d2 = d * d
    if kind == "adagrad":
        v.add_(d2)
    elif kind == "adam":
        v.mul_(beta2).add_((1.0 - beta2) * d2)
    elif kind == "yogi":
        v.sub_((1.0 - beta2) * d2 * torch.sign(v - d2))
    else:
        raise ValueError(f"unknown server optimizer {kind!r}")
    return theta.add_(lr * m / (v.sqrt() + tau))


def server_opt_apply(theta: torch.Tensor, models: torch.Tensor, weights: torch.Tensor, kind: str, lr: float, m=None, v=None,
                     beta1: float = 0.9, beta2: float = 0.99, tau: float = 1e-3, aggregator=None) -> torch.Tensor:
    """``avg = sum_k w_k models[k]`` (or the robust aggregate of ``aggregator``) then :func:`server_opt_step` (the oracle of
    the fused kernels)."""
    return server_opt_step(theta, aggregate(models, weights, aggregator, theta), kind, lr, m, v, beta1, beta2, tau)


# ------------------------------------------------------------------------------------------------
# uplink codec (ops/csrc/uplink_quant.cuh; fl/uplink.py)
# ------------------------------------------------------------------------------------------------
UQ_BLOCK = 256
_UQ_LEVELS = {8: 127, 4: 7}


def _fmix32(h: np.ndarray) -> np.ndarray:
    """MurmurHash3 finalizer on uint32 arrays (wrap-around arithmetic)."""
    h = h ^ (h >> np.uint32(16))
    h = h * np.uint32(0x85EBCA6B)
    h = h ^ (h >> np.uint32(13))
    h = h * np.uint32(0xC2B2AE35)
    return h ^ (h >> np.uint32(16))


def uplink_uniform(keys, n: int) -> np.ndarray:
    """float32 ``[K, n]``: r_j = (fmix32(key ^ (j * 0x9E3779B9)) >> 8) * 2^-24 for the elements j < n of every key."""
    keys = np.asarray(keys, dtype=np.int64).astype(np.uint32).reshape(-1, 1)
    with np.errstate(over="ignore"):
        j = np.arange(n, dtype=np.uint32) * np.uint32(0x9E3779B9)
        h = _fmix32(keys ^ j[None, :])
    return (h >> np.uint32(8)).astype(np.float32) * np.float32(2.0 ** -24)


def encode_delta(models: torch.Tensor, theta: torch.Tensor, bits: int, keys) -> Tuple[torch.Tensor, torch.Tensor]:
    """The int8 / int4 codes of ``models [K, P] - theta [P]`` rounded with the uint32 ``keys [K]``: ``(payload uint8 [K,
    payload bytes], scales float32 [K, ceil(P / 256)])`` in the wire layout (two's complement bytes, or nibbles with element
    2i in the low nibble of byte i).  Vectorised numpy; bit for bit what ``quantize_delta_kernel`` writes."""
    L = _UQ_LEVELS[bits]
    m = models.detach().to("cpu", torch.float32).reshape(len(keys), -1).numpy()
    t = theta.detach().to("cpu", torch.float32).reshape(-1).numpy()
    K, P = m.shape
    if P >= 1 << 31:
        raise ValueError("the codec indexes elements as uint32: P must be below 2^31")
    nblk = (P + UQ_BLOCK - 1) // UQ_BLOCK
    with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
        d = np.zeros((K, nblk * UQ_BLOCK), dtype=np.float32)
        d[:, :P] = m - t[None, :]
        db = d.reshape(K, nblk, UQ_BLOCK)
        sbits = (db.view(np.uint32) & np.uint32(0x7FFFFFFF)).max(axis=2)
        nonfinite = sbits >= np.uint32(0x7F800000)
        s = sbits.view(np.float32)
        inv = np.float32(L) / s
        zero = ~nonfinite & ~(inv <= np.finfo(np.float32).max)
        step = s / np.float32(L)
        dead = nonfinite | zero
        step = np.where(zero, np.float32(0.0), step)
        step = np.where(nonfinite, np.array(0x7FC00000, dtype=np.uint32).view(np.float32), step).astype(np.float32)
        inv = np.where(dead, np.float32(0.0), inv).astype(np.float32)
        u = (db * inv[:, :, None]).reshape(K, -1)
        f = np.floor(u)
        r = uplink_uniform(keys, nblk * UQ_BLOCK)
        q = f + (r < (u - f)).astype(np.float32)
        q = np.where(np.repeat(dead, UQ_BLOCK, axis=1), np.float32(0.0), q)
        q = np.clip(q, -L, L).astype(np.int8)[:, :P]
    if bits == 8:
        payload = q.view(np.uint8)
    else:
        nib = (q.astype(np.uint8) & np.uint8(0xF))
        if P % 2:
            nib = np.concatenate([nib, np.zeros((K, 1), dtype=np.uint8)], axis=1)
        payload = nib[:, 0::2] | (nib[:, 1::2] << np.uint8(4))
    return torch.from_numpy(np.ascontiguousarray(payload)), torch.from_numpy(np.ascontiguousarray(step))


def decode_codes(payload: torch.Tensor, bits: int, n: int) -> torch.Tensor:
    """int32 codes ``[K, n]`` of a payload in the wire layout (rows may carry trailing padding)."""
    b = payload.detach().to("cpu").numpy().astype(np.uint8)
    if bits == 8:
        q = b[:, :n].view(np.int8).astype(np.int32)
    else:
        b = b[:, :(n + 1) // 2]
        nib = np.stack([b & np.uint8(0xF), b >> np.uint8(4)], axis=2).reshape(b.shape[0], -1)[:, :n].astype(np.int32)
        q = np.where(nib >= 8, nib - 16, nib)
    return torch.from_numpy(np.ascontiguousarray(q))


def decode_delta(payload: torch.Tensor, scales: torch.Tensor, bits: int, n: int) -> torch.Tensor:
    """float32 deltas ``[K, n]``: d^_j = (float)q_j * step of j's block."""
    q = decode_codes(payload, bits, n).float()
    step = scales.detach().to("cpu", torch.float32).repeat_interleave(UQ_BLOCK, dim=1)[:, :n]
    return q * step


def fedavg_apply_quantized(theta: torch.Tensor, payload: torch.Tensor, scales: torch.Tensor, weights: torch.Tensor, bits: int,
                           server_lr: float = 1.0, opt=None, aggregator=None) -> torch.Tensor:
    """``a = theta + aggregate(decoded deltas)`` (the weighted sum, or the robust aggregate of ``aggregator``), then
    ``theta += server_lr (a - theta)`` or the server optimizer step of ``opt`` (a ``ServerOptState``), in place."""
    deltas = decode_delta(payload, scales, bits, theta.numel()).to(theta.device)
    w = weights.to(theta.device, torch.float32) if weights is not None else None
    avg = theta + aggregate(deltas, w, aggregator, torch.zeros_like(theta).reshape(-1))
    if opt is None:
        return theta.add_(server_lr * (avg - theta))
    b1, b2, tau = opt.hyper
    return server_opt_step(theta, avg, opt.kind, opt.lr, opt.m, opt.v, b1, b2, tau)


# ------------------------------------------------------------------------------------------------
# top-k uplink with error feedback (ops/csrc/uplink_topk.cuh; fl/uplink.py)
# ------------------------------------------------------------------------------------------------
def topk_entries(p: int, k: int) -> int:
    """E(P, k) = k (nblk - 1) + min(k, m_last): the entries of one row."""
    nblk = (p + UQ_BLOCK - 1) // UQ_BLOCK
    return k * (nblk - 1) + min(k, p - (nblk - 1) * UQ_BLOCK)


def topk_keys(v: np.ndarray) -> np.ndarray:
    """uint32 selection keys of float32 ``v``: the bits of |v|, every NaN mapped to 0x7f800001."""
    a = v.view(np.uint32) & np.uint32(0x7FFFFFFF)
    return np.where(a > np.uint32(0x7F800000), np.uint32(0x7F800001), a)


def encode_topk_delta(models: torch.Tensor, theta: torch.Tensor, residual: torch.Tensor, k: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """The top-``k`` entries per 256-element block of ``v = (models [K, P] - theta [P]) + residual [K, P]``: ``(indices
    uint8 [K, E], values float32 [K, E])`` in the wire layout (offsets ascending inside each block, blocks packed), and
    ``residual`` overwritten in place with ``v`` minus the sent entries.  Vectorised numpy; bit for bit what
    ``topk_delta_kernel`` writes (up to NaN payloads, which the GPU makes canonical)."""
    if not 1 <= k <= 32:
        raise ValueError(f"topk keeps 1..32 entries per block, not {k}")
    m = models.detach().to("cpu", torch.float32).reshape(residual.shape).numpy()
    t = theta.detach().to("cpu", torch.float32).reshape(-1).numpy()
    e = residual.detach().to("cpu", torch.float32).numpy()
    with np.errstate(over="ignore", invalid="ignore"):
        v = (m - t[None, :]) + e
    idx, pos = _topk_select(v, k)
    values = np.take_along_axis(v, pos, axis=1)
    rest = v.copy()
    np.put_along_axis(rest, pos, np.float32(0.0), axis=1)
    residual.copy_(torch.from_numpy(rest))
    return torch.from_numpy(np.ascontiguousarray(idx.astype(np.uint8))), torch.from_numpy(np.ascontiguousarray(values))


def _topk_select(v: np.ndarray, k: int) -> Tuple[np.ndarray, np.ndarray]:
    """The wire offsets ``[K, E]`` of the top-``k`` selection of every 256-element block of float32 ``v [K, P]`` and their
    positions in ``v`` (int64)."""
    K, P = v.shape
    nblk = (P + UQ_BLOCK - 1) // UQ_BLOCK
    # composite = key 256 + (255 - offset): unique inside a block, greater = kept first (the lower offset wins a tie);
    # elements past P get key -1 and are kept only in a last block shorter than k, where they are cut off below
    key = np.full((K, nblk * UQ_BLOCK), -1, dtype=np.int64)
    key[:, :P] = topk_keys(v)
    comp = key.reshape(K, nblk, UQ_BLOCK) * UQ_BLOCK + (UQ_BLOCK - 1 - np.arange(UQ_BLOCK, dtype=np.int64))
    top = -np.sort(-comp, axis=2)[:, :, :k]
    off = np.sort((UQ_BLOCK - 1) - (top & (UQ_BLOCK - 1)), axis=2)
    idx = off.reshape(K, nblk * k)[:, :topk_entries(P, k)]
    return idx, _topk_positions(idx, k)


def _topk_positions(idx: np.ndarray, k: int) -> np.ndarray:
    """element positions (int64) of the wire offsets ``idx [K, E]``: block ``e // k`` of entry ``e``"""
    return idx.astype(np.int64) + (np.arange(idx.shape[1]) // k * UQ_BLOCK)[None, :]


def decode_topk_delta(indices: torch.Tensor, values: torch.Tensor, k: int, n: int) -> torch.Tensor:
    """float32 deltas ``[K, n]``: the entries at their positions, zero elsewhere."""
    idx = indices.detach().to("cpu").numpy().astype(np.int64)
    pos = idx + (np.arange(idx.shape[1]) // k * UQ_BLOCK)[None, :]
    out = np.zeros((idx.shape[0], n), dtype=np.float32)
    np.put_along_axis(out, pos, values.detach().to("cpu", torch.float32).numpy(), axis=1)
    return torch.from_numpy(out)


def fedavg_apply_topk(theta: torch.Tensor, indices: torch.Tensor, values: torch.Tensor, weights: torch.Tensor, k: int,
                      server_lr: float = 1.0, opt=None) -> torch.Tensor:
    """``a = theta + sum_k w_k (decoded sparse delta k)``, then ``theta += server_lr (a - theta)`` or the server optimizer
    step of ``opt`` (a ``ServerOptState``), in place."""
    deltas = decode_topk_delta(indices, values, k, theta.numel()).to(theta.device)
    avg = theta + fedavg_flat(deltas, weights.to(theta.device, torch.float32))
    if opt is None:
        return theta.add_(server_lr * (avg - theta))
    b1, b2, tau = opt.hyper
    return server_opt_step(theta, avg, opt.kind, opt.lr, opt.m, opt.v, b1, b2, tau)


# ------------------------------------------------------------------------------------------------
# compressed downlink (ops/csrc/downlink.cuh; fl/uplink.py)
# ------------------------------------------------------------------------------------------------
def _replica_np(replica: torch.Tensor) -> np.ndarray:
    if replica.dtype != torch.float32 or not replica.is_contiguous():
        raise ValueError("the replica must be a contiguous float32 tensor (it is updated in place)")
    return replica.detach().to("cpu").reshape(-1).numpy().copy()


def encode_downlink(theta: torch.Tensor, replica: torch.Tensor, codec, key: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """The downlink wire of ``theta [P] - replica [P]`` and ``replica`` advanced in place by what it carries: int8 / int4
    ``(payload uint8 [codec.payload_bytes(P)], scales float32 [codec.scale_count(P)])`` rounded with the uint32 ``key``
    (``encode_delta``'s codes, then ``r += q step`` in fp32), or topk ``(indices uint8 [E], values float32 [E])`` of ``v =
    theta - replica`` (``encode_topk_delta``'s selection, then ``r += v`` at the sent entries).  Bit for bit what
    ``downlink_quant_kernel`` / ``downlink_topk_kernel`` write (up to NaN payloads)."""
    r = _replica_np(replica)
    t = theta.detach().to("cpu", torch.float32).reshape(-1)
    if codec.quantized:
        payload, scales = encode_delta(t.view(1, -1), torch.from_numpy(r), codec.bits, [key])
        apply_downlink(replica, payload[0], scales[0], codec)
        return payload[0], scales[0]
    if not codec.sparse:
        raise ValueError("encode_downlink needs an int8 / int4 / topk codec")
    if not 1 <= codec.k <= 32:
        raise ValueError(f"topk keeps 1..32 entries per block, not {codec.k}")
    with np.errstate(over="ignore", invalid="ignore"):
        v = t.numpy() - r
    idx, pos = _topk_select(v[None, :], codec.k)
    values = v[pos[0]]
    with np.errstate(over="ignore", invalid="ignore"):
        r[pos[0]] = r[pos[0]] + values
    replica.copy_(torch.from_numpy(r).view_as(replica))
    return torch.from_numpy(np.ascontiguousarray(idx[0].astype(np.uint8))), torch.from_numpy(np.ascontiguousarray(values))


def apply_downlink(replica: torch.Tensor, a: torch.Tensor, b: torch.Tensor, codec) -> torch.Tensor:
    """``replica [P]`` advanced in place by a downlink wire: int8 / int4 ``(a, b) = (payload, scales)``, ``r += q step``; topk
    ``(a, b) = (indices, values)``, ``r += value`` at each entry's position.  Bit for bit what ``replica_apply_q_kernel`` /
    ``replica_apply_topk_kernel`` write."""
    r = _replica_np(replica)
    with np.errstate(over="ignore", invalid="ignore"):
        if codec.quantized:
            r = r + decode_delta(a.reshape(1, -1), b.reshape(1, -1), codec.bits, r.size)[0].numpy()
        elif codec.sparse:
            pos = _topk_positions(a.detach().to("cpu").numpy().reshape(1, -1), codec.k)[0]
            r[pos] = r[pos] + b.detach().to("cpu", torch.float32).numpy().reshape(-1)
        else:
            raise ValueError("apply_downlink needs an int8 / int4 / topk codec")
    return replica.copy_(torch.from_numpy(r).view_as(replica))


# ------------------------------------------------------------------------------------------------
# secure aggregation (ops/csrc/secagg.cuh; fl/secagg.py)
# ------------------------------------------------------------------------------------------------
SA_WORDS = 16
SA_MAX_ELEMS = 1 << 36
_SIGMA = (0x61707865, 0x3320646E, 0x79622D32, 0x6B206574)
_DIAG = ((0, 4, 8, 12), (1, 5, 9, 13), (2, 6, 10, 14), (3, 7, 11, 15), (0, 5, 10, 15), (1, 6, 11, 12), (2, 7, 8, 13), (3, 4, 9, 14))


def _rotl(x: np.ndarray, r: int) -> np.ndarray:
    return (x << np.uint32(r)) | (x >> np.uint32(32 - r))


def _chacha(keys: np.ndarray, counters: np.ndarray, nonce=(0, 0, 0)) -> np.ndarray:
    """uint32 ``[S, N, 16]``: the ChaCha20 blocks (RFC 8439 §2.3) of the keys ``[S, 8]`` at the block counters ``[N]``."""
    S, N = keys.shape[0], counters.size
    init = [np.full((S, N), c, dtype=np.uint32) for c in _SIGMA]
    init += [np.repeat(keys[:, i:i + 1].astype(np.uint32), N, axis=1) for i in range(8)]
    init += [np.repeat(counters.astype(np.uint32)[None, :], S, axis=0)]
    init += [np.full((S, N), w, dtype=np.uint32) for w in nonce]
    x = [w.copy() for w in init]
    for _ in range(10):
        for a, b, c, d in _DIAG:
            x[a] += x[b]; x[d] ^= x[a]; x[d] = _rotl(x[d], 16)   # noqa: E702
            x[c] += x[d]; x[b] ^= x[c]; x[b] = _rotl(x[b], 12)   # noqa: E702
            x[a] += x[b]; x[d] ^= x[a]; x[d] = _rotl(x[d], 8)    # noqa: E702
            x[c] += x[d]; x[b] ^= x[c]; x[b] = _rotl(x[b], 7)    # noqa: E702
    return np.stack([x[i] + init[i] for i in range(16)], axis=2)


def _key_words(keys) -> np.ndarray:
    """uint32 ``[S, 8]`` of 32-byte keys (bytes), or of an int32 / uint32 ``[S, 8]`` tensor / array of their words"""
    if isinstance(keys, torch.Tensor):
        return keys.detach().to("cpu").contiguous().view(torch.int32).numpy().view(np.uint32).reshape(-1, 8)
    if isinstance(keys, np.ndarray):
        return keys.view(np.uint32).reshape(-1, 8)
    keys = list(keys)
    if any(not isinstance(k, (bytes, bytearray)) or len(k) != 32 for k in keys):
        raise ValueError("stream keys are 32 bytes each")
    return np.frombuffer(b"".join(keys), dtype="<u4").astype(np.uint32).reshape(-1, 8)


def chacha20_blocks(key: bytes, counter: int, count: int, nonce: bytes = bytes(12)) -> np.ndarray:
    """uint32 ``[count, 16]``: the ChaCha20 blocks ``counter .. counter + count - 1`` of the 32-byte ``key`` and 12-byte
    ``nonce`` (RFC 8439 §2.3; serialised little-endian they are the keystream of §2.4)."""
    n = np.frombuffer(bytes(nonce), dtype="<u4")
    return _chacha(_key_words([bytes(key)]), np.arange(counter, counter + count, dtype=np.uint64).astype(np.uint32), tuple(int(w) for w in n))[0]


def secagg_streams(keys, signs, n: int) -> np.ndarray:
    """uint32 ``[n]``: ``sum_s signs[s] PRG(keys[s])`` (mod 2^32), element ``e`` of a stream being word ``e mod 16`` of its
    block ``e / 16`` with nonce 0."""
    kw = _key_words(keys)
    sg = np.asarray(signs.cpu() if isinstance(signs, torch.Tensor) else signs, dtype=np.int64).reshape(-1)
    if sg.size != kw.shape[0] or not np.isin(sg, (-1, 1)).all():
        raise ValueError("one sign (+1 / -1) per stream key")
    if n >= SA_MAX_ELEMS:
        raise ValueError("a stream indexes blocks with one uint32 word: P must be below 2^36")
    cols = (n + SA_WORDS - 1) // SA_WORDS
    counters = np.arange(cols, dtype=np.uint64).astype(np.uint32)
    acc = np.zeros(cols * SA_WORDS, dtype=np.uint32)
    step = max(1, (1 << 21) // max(1, cols))               # streams per chunk: bounded temporaries
    for s0 in range(0, kw.shape[0], step):
        blocks = _chacha(kw[s0:s0 + step], counters).reshape(-1, cols * SA_WORDS)
        neg = sg[s0:s0 + step] < 0
        acc += blocks[~neg].sum(axis=0, dtype=np.uint32) - blocks[neg].sum(axis=0, dtype=np.uint32)
    return acc[:n]


def secagg_encode(delta: np.ndarray, clip: float, frac_bits: int) -> Tuple[np.ndarray, int, int]:
    """``(q uint32 [P], clipped, nonfinite)``: the fixed-point codes of float32 deltas (``sa_encode``)."""
    d = np.asarray(delta, dtype=np.float32).reshape(-1)
    c32 = np.float32(clip)
    with np.errstate(invalid="ignore"):
        nan, inf = np.isnan(d), np.isinf(d)
        clipped = int((~nan & ~inf & (np.abs(d) > c32)).sum())
        c = np.where(nan, np.float32(0.0), np.clip(d, -c32, c32)).astype(np.float32)
    q = np.rint(c * np.float32(2.0 ** frac_bits)).astype(np.int64).astype(np.int32)
    return q.view(np.uint32), clipped, int(nan.sum() + inf.sum())


def secagg_mask(model: torch.Tensor, theta: torch.Tensor, keys, signs, clip: float, frac_bits: int) -> Tuple[torch.Tensor, int, int]:
    """A device's masked update: ``(y uint32 [P], clipped, nonfinite)`` with ``y = enc(model - theta) + sum_s signs[s]
    PRG(keys[s])`` (mod 2^32).  Bit for bit what ``secagg_mask_kernel`` writes."""
    m = model.detach().to("cpu", torch.float32).reshape(-1).numpy()
    t = theta.detach().to("cpu", torch.float32).reshape(-1).numpy()
    with np.errstate(invalid="ignore", over="ignore"):
        q, clipped, nonfinite = secagg_encode(m - t, clip, frac_bits)
    return torch.from_numpy(q + secagg_streams(keys, signs, q.size)), clipped, nonfinite


def secagg_unmask_sum(masked: torch.Tensor, keys, signs) -> np.ndarray:
    """uint32 ``[P]``: the sum of the masked rows ``[K, P]`` plus the signed correction streams (mod 2^32)."""
    y = masked.detach().to("cpu").contiguous().view(torch.int32).numpy().view(np.uint32)
    y = y.reshape(-1, y.shape[-1])
    return y.sum(axis=0, dtype=np.uint32) + secagg_streams(keys, signs, y.shape[1])


def secagg_decode(z: np.ndarray, frac_bits: int, n: int) -> np.ndarray:
    """float32 mean of ``n`` survivors whose codes sum to ``z`` (``sa_decode``)."""
    zf = np.asarray(z, dtype=np.uint32).view(np.int32).astype(np.float32)
    return (zf * np.float32(2.0 ** -frac_bits)) / np.float32(n)


def _fmaf(a, b, c) -> np.ndarray:
    """float32 fused multiply-add: the float32 product is exact in float64, then one float64 add and the float32 rounding"""
    f = lambda x: np.asarray(x, dtype=np.float64)  # noqa: E731 - (a one-element array stays an array)
    return (f(a) * f(b) + f(c)).astype(np.float32)


def _server_opt_np(t: np.ndarray, a: np.ndarray, opt, server_lr: float) -> np.ndarray:
    """``server_opt.cuh``'s step of theta towards ``a`` in float32 numpy with its fmaf; the moments of ``opt`` updated in place"""
    f = np.float32
    if opt is None or opt.kind == "sgd":
        return _fmaf(f(server_lr if opt is None else opt.lr), a - t, t)
    lr = f(opt.lr)
    b1, b2, tau = (f(h) for h in opt.hyper)
    d = a - t
    m = opt.m.detach().cpu().numpy().astype(np.float32)
    if opt.kind == "avgm":
        m = _fmaf(b1, m, d)
        opt.m.copy_(torch.from_numpy(m))
        return _fmaf(lr, m, t)
    m = _fmaf(b1, m, (f(1.0) - b1) * d)
    v = opt.v.detach().cpu().numpy().astype(np.float32)
    d2 = d * d
    if opt.kind == "adagrad":
        v = _fmaf(d, d, v)
    elif opt.kind == "adam":
        v = _fmaf(b2, v, (f(1.0) - b2) * d2)
    elif opt.kind == "yogi":
        s = np.where(v > d2, f(1.0), np.where(v < d2, f(-1.0), f(0.0)))
        v = _fmaf(-(f(1.0) - b2) * s, d2, v)
    else:
        raise ValueError(f"unknown server optimizer {opt.kind!r}")
    opt.m.copy_(torch.from_numpy(m))
    opt.v.copy_(torch.from_numpy(v))
    return _fmaf(lr, m / (np.sqrt(v) + tau), t)


def fedavg_apply_secagg(theta: torch.Tensor, masked: torch.Tensor, keys, signs, frac_bits: int, n: int, server_lr: float = 1.0,
                        opt=None) -> torch.Tensor:
    """``mean = secagg_decode(secagg_unmask_sum(masked, keys, signs))``, ``a = theta + mean``, then ``theta += server_lr (a -
    theta)`` or the server optimizer step of ``opt`` (a ``ServerOptState``), in place; the float32 roundings of
    ``fedavg_secagg_kernel`` (fmaf where it has one): bit for bit what it writes."""
    mean = secagg_decode(secagg_unmask_sum(masked, keys, signs), frac_bits, n)
    t = theta.detach().to("cpu", torch.float32).reshape(-1).numpy()
    with np.errstate(over="ignore", invalid="ignore"):
        out = _server_opt_np(t, t + mean, opt, server_lr)
    return theta.copy_(torch.from_numpy(out).view_as(theta))


def based_deltas(models: torch.Tensor, ring: torch.Tensor, base_slot) -> torch.Tensor:
    """float32 ``[K, P]``: ``models[k] - ring[base_slot[k]]``, every row's delta to the global version it was trained from"""
    r = ring.detach().to("cpu", torch.float32)
    x = models.detach().to("cpu", torch.float32)[:, :r.shape[1]]
    return x - r[torch.as_tensor([int(b) for b in base_slot], dtype=torch.long)]


def fedavg_apply_based(theta: torch.Tensor, models: torch.Tensor, ring: torch.Tensor, base_slot, weights: torch.Tensor, write_slot: int,
                       server_lr: float = 1.0, opt=None, aggregator=None) -> torch.Tensor:
    """Asynchronous buffered aggregation's apply (``ROWS_F32_BASED``): the deltas ``d_k = models[k] - ring[base_slot[k]]``,
    ``a = theta + acc`` with ``acc = sum_k fmaf(w_k, d_k, acc)`` in row order from +0 (or the robust aggregate of the deltas:
    coordinate-wise unweighted, distance-based from 0 with ``weights`` as alpha), then ``theta += server_lr (a - theta)`` or
    the server optimizer step of ``opt``, in place; the new theta is also written to ``ring[write_slot]``.  The float32
    roundings of ``fedavg_based_kernel`` / the robust body: bit for bit what they write (the distance-based kinds within
    the tolerance of :func:`distance_aggregate`)."""
    d = based_deltas(models, ring, base_slot)
    t = theta.detach().to("cpu", torch.float32).reshape(-1).numpy()
    if aggregator is None or not aggregator.robust:
        w = weights.detach().to("cpu", torch.float32).numpy()
        acc = np.zeros_like(t)
        for k, dk in enumerate(d.numpy()):
            acc = _fmaf(w[k], dk, acc)
    elif aggregator.distance_based:
        acc = distance_aggregate(d, weights, aggregator, torch.zeros(d.shape[1]))[0].numpy()
    else:
        acc = robust_aggregate(d, None, aggregator.kind, aggregator.trim).numpy()
    with np.errstate(over="ignore", invalid="ignore"):
        out = torch.from_numpy(_server_opt_np(t, t + acc, opt, server_lr))
    ring[int(write_slot)].copy_(out.to(ring.device))
    return theta.copy_(out.view_as(theta).to(theta.device))


def linear_bias_relu(x, w, b, relu=True):
    y = x.float() @ w.float().t() + b.float()
    return torch.relu(y) if relu else y


def eval_binary(out: torch.Tensor, y: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """(sum of per-sample BCE, number of correct ``round(out)`` predictions) — cf.py:233-253."""
    y = y.reshape(out.shape).to(out.dtype)
    logp = torch.clamp(torch.log(out), min=-100.0)
    log1mp = torch.clamp(torch.log1p(-out), min=-100.0)
    loss = -(y * logp + (1 - y) * log1mp).sum()
    correct = (torch.round(out) == y).sum()
    return loss, correct


def argmax_rows(out: torch.Tensor) -> torch.Tensor:
    return out.argmax(1, keepdim=True)


def eval_summary_limits(classes: int, bins: int, threshold: float, rows: int = 0) -> None:
    """The limits of ``ops/csrc/eval_summary.cuh``: ValueError with the reason outside them"""
    if rows >= 1 << 32:
        raise ValueError(f"eval_summary: {rows} rows, at most 2^32 - 1 per call (the kernel counts in uint32 shared memory)")
    if not 1 <= classes <= 32:
        raise ValueError(f"eval_summary: {classes} output columns, the summary takes 1 to 32")
    if bins < 2 or bins > 4096 or bins & (bins - 1):
        raise ValueError(f"eval_summary: bins must be a power of two in [2, 4096], not {bins}")
    if classes * 2 * bins > 32768:
        raise ValueError(f"eval_summary: {classes} histograms of 2 x {bins} bins exceed the 32768 counters of one summary")
    if not 0.0 <= threshold <= 1.0:
        raise ValueError(f"eval_summary: the threshold must be in [0, 1], not {threshold}")


def eval_summary(scores: torch.Tensor, labels: torch.Tensor, bins: int = 256, threshold: float = 0.5,
                 offsets: Optional[Sequence[int]] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """PyTorch transcription of ``ops/csrc/eval_summary.cuh``: ``(counts int64 [S, L], loss_sum float64 [S])`` of the rows
    ``offsets[s] .. offsets[s + 1]`` of ``scores [N, C]`` / ``labels [N]`` (one segment of all rows when ``offsets`` is None).
    The loss sums its 2048-row chunks in chunk order (inside a chunk torch's own order: equal to the kernel's to ~1e-15)."""
    scores = scores.detach().float().cpu()
    scores = scores.view(-1, 1) if scores.dim() == 1 else scores
    n, c = scores.shape
    eval_summary_limits(c, bins, threshold, n)
    y = labels.detach().float().cpu().reshape(-1)
    offsets = [0, n] if offsets is None else [int(o) for o in offsets]
    cp = 2 if c == 1 else c
    conf0, hist0 = 2, 2 + cp * cp
    length = hist0 + c * 2 * bins
    lab_ok = (y >= 0) & (y < cp) & (y == torch.floor(y))
    if c == 1:
        p = scores[:, 0]
        valid = (p >= 0) & (p <= 1) & lab_ok
        p = torch.where(valid, p, torch.zeros_like(p))
        yi = torch.where(valid, y, torch.zeros_like(y)).long()
        pd = p.double()
        row_loss = torch.where(yi == 1, -torch.log(pd).clamp(min=-100.0), -torch.log1p(-pd).clamp(min=-100.0))
        b = (p * float(bins)).long().clamp(max=bins - 1)
        words = [conf0 + 2 * yi + (p > threshold).long(), hist0 + yi * bins + b]
    else:
        valid = torch.isfinite(scores).all(1) & lab_ok
        z = torch.where(valid[:, None], scores, torch.zeros_like(scores))
        yi = torch.where(valid, y, torch.zeros_like(y)).long()
        m, arg = z.max(1).values, z.argmax(1)
        e = torch.exp(z.double() - m.double()[:, None])
        s = e[:, 0].clone()
        for k in range(1, c):
            s = s + e[:, k]
        row_loss = torch.log(s) - (z.double().gather(1, yi[:, None])[:, 0] - m.double())
        b = ((e / s[:, None]) * float(bins)).long().clamp(max=bins - 1)
        cls = torch.arange(c)
        words = [conf0 + c * yi + arg] + [hist0 + (2 * k + (yi == k).long()) * bins + b[:, k] for k in cls.tolist()]
    row_loss = torch.where(valid, row_loss, torch.zeros_like(row_loss))
    counts = torch.zeros(len(offsets) - 1, length, dtype=torch.int64)
    loss = torch.zeros(len(offsets) - 1, dtype=torch.float64)
    for s_idx, (lo, hi) in enumerate(zip(offsets[:-1], offsets[1:])):
        if lo > hi or lo < 0 or hi > n:
            raise ValueError("offsets must rise from 0 to N")
        v = valid[lo:hi]
        counts[s_idx, 0] = hi - lo
        counts[s_idx, 1] = int((~v).sum())
        for w in words:
            counts[s_idx] += torch.bincount(w[lo:hi][v], minlength=length)
        total = 0.0
        for q in range(lo, hi, 2048):
            total += float(row_loss[q:min(q + 2048, hi)].sum())
        loss[s_idx] = total
    if offsets[0] != 0 or offsets[-1] != n:
        raise ValueError("offsets must rise from 0 to N")
    return counts, loss


def recon_summary_limits(dim: int, bins: int, rows: int = 0, alarm_bin: Optional[int] = None) -> None:
    """The limits of ``ops/csrc/recon_summary.cuh``: ValueError with the reason outside them"""
    if rows >= 1 << 32:
        raise ValueError(f"recon_summary: {rows} rows, at most 2^32 - 1 per call (the kernel counts in uint32 shared memory)")
    if not 1 <= dim <= 1024:
        raise ValueError(f"recon_summary: {dim} columns, the summary takes 1 to 1024")
    if bins < 32 or bins > 4096 or bins & (bins - 1):
        raise ValueError(f"recon_summary: bins must be a power of two in [32, 4096], not {bins}")
    if alarm_bin is not None and not 0 <= alarm_bin <= bins:
        raise ValueError(f"recon_summary: the alarm bin must be in [0, {bins}], not {alarm_bin}")


def recon_bin(e: torch.Tensor, bins: int) -> torch.Tensor:
    """``rs_bin`` of ``recon_summary.cuh``: the bin of every float64 error, from the bits of ``(float)e`` (int64)"""
    sub = (bins // 32).bit_length() - 1
    u = e.float().view(torch.int32).long() & 0xFFFFFFFF
    b = (((u >> 23) - 103) << sub) + ((u & 0x7FFFFF) >> (23 - sub))
    return torch.where(u < 0x33800000, torch.zeros_like(b), torch.where(u >= 0x43800000, torch.full_like(b, bins - 1), b))


def recon_summary(xhat: torch.Tensor, x: torch.Tensor, labels: Optional[torch.Tensor] = None, bins: int = 256,
                  offsets: Optional[Sequence[int]] = None, alarm_bin: Optional[int] = None):
    """PyTorch transcription of ``ops/csrc/recon_summary.cuh``, equal to the kernel bit for bit: ``(counts int64 [S, 2 + 2 B],
    err_sum float64 [S], err fp32 [N] or None, flag uint8 [N] or None)`` of the rows ``offsets[s] .. offsets[s + 1]`` (one
    segment of all rows when ``offsets`` is None); the per-row outputs only with ``alarm_bin``.  The error sum follows the
    kernel's order exactly: 2048-row chunks, thread t adding rows t, t + 256, ..., t + 1792, a xor butterfly over each warp's
    32 lanes, the 8 warp sums in order, the chunk sums in order."""
    xhat = xhat.detach().float().cpu()
    x = x.detach().float().cpu()
    if xhat.dim() != 2 or xhat.shape != x.shape:
        raise ValueError("xhat and x must both be [N, D]")
    n, d = x.shape
    recon_summary_limits(d, bins, n, alarm_bin)
    offsets = [0, n] if offsets is None else [int(o) for o in offsets]
    if len(offsets) < 2 or offsets[0] != 0 or offsets[-1] != n or any(b < a for a, b in zip(offsets[:-1], offsets[1:])):
        raise ValueError("offsets must rise from 0 to N")
    dd = (xhat - x).double()                                        # d formed in fp32, d^2 exact in float64
    sq = dd * dd
    e = torch.zeros(n, dtype=torch.float64)
    for c in range(d):
        e = e + sq[:, c]
    valid = torch.isfinite(xhat).all(1) & torch.isfinite(x).all(1)
    y = torch.zeros(n, dtype=torch.int64)
    if labels is not None:
        lab = labels.detach().float().cpu().reshape(-1)
        y = torch.where(lab == 0, 0, torch.where(lab == 1, 1, -1)).long()
        valid &= y >= 0
    b = recon_bin(e, bins)
    words = torch.where(valid, 2 + y.clamp(min=0) * bins + b, torch.zeros_like(b))
    ev = torch.where(valid, e, torch.zeros_like(e))
    length = 2 + 2 * bins
    counts = torch.zeros(len(offsets) - 1, length, dtype=torch.int64)
    total = torch.zeros(len(offsets) - 1, dtype=torch.float64)
    for s_idx, (lo, hi) in enumerate(zip(offsets[:-1], offsets[1:])):
        v = valid[lo:hi]
        counts[s_idx, 0] = hi - lo
        counts[s_idx, 1] = int((~v).sum())
        counts[s_idx] += torch.bincount(words[lo:hi][v], minlength=length)
        chunks = (hi - lo + 2047) // 2048
        if chunks == 0:
            continue
        pad = torch.zeros(chunks * 2048, dtype=torch.float64)
        pad[:hi - lo] = ev[lo:hi]
        rows = pad.view(chunks, 8, 256)                              # [chunk, i, thread]
        acc = rows[:, 0]
        for i in range(1, 8):
            acc = acc + rows[:, i]
        lanes = acc.view(chunks, 8, 32)                              # [chunk, warp, lane]
        for o in (16, 8, 4, 2, 1):
            lanes = lanes[..., :o] + lanes[..., o:2 * o]
        warps = lanes[..., 0]
        part = warps[:, 0]
        for w in range(1, 8):
            part = part + warps[:, w]
        t = torch.zeros((), dtype=torch.float64)
        for q in range(chunks):
            t = t + part[q]
        total[s_idx] = t
    err = flag = None
    if alarm_bin is not None:
        err = e.float()
        flag = ((~valid) | (b >= alarm_bin)).to(torch.uint8)
    return counts, total, err, flag
