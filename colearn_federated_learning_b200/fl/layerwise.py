"""Layer-wise local training of wide MLPs on wgmma GEMMs (BASELINE config 5, SURVEY K7/K8/K12).

Every Linear of the wide MLP (10 → 4096×4 → 2) runs on ``ops.gemm_bf16`` — the hand-written
wgmma/TMA kernel — in three roles that all reduce to ``C = A·Bᵀ`` with K-major operands:

    forward   H_l  = relu(H_{l-1} · W_lᵀ + b_l)       A = H_{l-1}[B,in]   B = W_l[out,in]   (+bias, relu)
    dgrad     dZ_{l-1} = (dZ_l · W_l) ⊙ relu'          A = dZ_l[B,out]     B = W_lᵀ[in,out]  (+mask, +colsum = db)
    wgrad     W_l ← W_l − lr · dZ_lᵀ · H_{l-1}         A = dZ_lᵀ[out,B]    B = H_{l-1}ᵀ[in,B] (+fused SGD on the
                                                        fp32 master, bf16 shadows W / Wᵀ refreshed in the epilogue)

The transposed activations / gradients the wgrad needs are written by the producing epilogues
(``out_bf16_t``), the bias gradient is the post-mask column sum of the dgrad epilogue, the SGD
step never materialises dW.  fp32 master weights live in the flat arena (what FedAvg
averages); bf16 shadows of the three 4096×4096 layers are *views into the bf16 shadow arena* that
the two-shot FedAvg kernel fills over NVLink, so the first forward GEMM of a round can poll the
per-chunk ready flags and start on the rows that have landed (fused broadcast → GEMM, SURVEY K1).
The 10-wide input and 2-wide head are zero-padded to tile multiples (128).
"""
from __future__ import annotations

import os
from typing import Dict, List, Optional, Tuple

import torch

from .. import ops
from ..ops import conv as conv_ops
from ..models import MLPSpec

PAD = 128


class ReadySpec:
    """Where the two-shot broadcast publishes per-chunk readiness (fused broadcast -> GEMM, SURVEY K1).
    ``epoch_ptr`` (device uint32) takes precedence over ``epoch`` so a captured CUDA graph can be replayed
    every round with a new epoch."""

    def __init__(self, flags_ptr: int, chunk_elems: int, epoch: int = 0, epoch_ptr: int = 0) -> None:
        self.flags_ptr, self.chunk_elems, self.epoch, self.epoch_ptr = int(flags_ptr), int(chunk_elems), int(epoch), int(epoch_ptr)


def _pad_to(n: int, m: int = PAD) -> int:
    return (n + m - 1) // m * m


class LayerwiseMLPTrainer:
    _cache: Dict[Tuple, "LayerwiseMLPTrainer"] = {}

    @staticmethod
    def supports(spec: MLPSpec, cfg) -> bool:
        """Any MLP with at least one hidden layer: widths that are not multiples of 128 are zero-padded (a padded hidden
        neuron has zero weights and bias, outputs relu(0) = 0 and receives a zero gradient through the ReLU mask), batches
        that are not are padded with rows whose loss gradient is zero (:meth:`forward`), so the 128-row GEMM tiles always
        see full operands.  Losses: softmax cross-entropy on a linear head, BCE / SSE / MSE on a sigmoid or linear head."""
        hidden = spec.dims[1:-1]
        if len(hidden) < 1 or cfg.batch_size < 1:
            return False
        if cfg.loss == "xent":
            return spec.out_activation == "none"
        if cfg.loss == "bce":
            return spec.out_activation == "sigmoid"
        return cfg.loss in ("sse", "mse") and spec.out_activation in ("none", "sigmoid")

    @staticmethod
    def supports_fused(spec: MLPSpec, cfg) -> bool:
        """The stricter shape the fused-broadcast / CUDA-graph round of the engine is built for: every hidden layer and the
        batch fill whole 128-wide tiles, cross-entropy head (BASELINE config 5)."""
        hidden = spec.dims[1:-1]
        return (len(hidden) >= 1 and all(h % 128 == 0 for h in hidden) and cfg.batch_size % 128 == 0
                and cfg.loss == "xent" and spec.out_activation == "none")

    @classmethod
    def cached(cls, spec: MLPSpec, flat: torch.Tensor, batch_size: int) -> "LayerwiseMLPTrainer":
        key = (spec.dims, flat.data_ptr(), batch_size)
        tr = cls._cache.get(key)
        if tr is None:
            if len(cls._cache) > 4:
                cls._cache.clear()
            tr = cls._cache[key] = cls(spec, flat, batch_size)
        return tr

    def __init__(self, spec: MLPSpec, flat: torch.Tensor, batch_size: int, shadow: Optional[torch.Tensor] = None,
                 dgrad_kn: Optional[bool] = None, wgrad_mn: Optional[bool] = None) -> None:
        # b = the caller's batch size, B = rows of every activation / gradient matrix (whole 128-row tiles); rows >= b carry a
        # zero loss gradient, so they take part in no update
        self.spec, self.b, self.B, self.dev = spec, int(batch_size), _pad_to(int(batch_size)), flat.device
        self._dz_rows = 0                                      # rows of dz[L-1] written since it was last all-zero
        # default (COLEARN_MLP_DGRAD_KN=0 restores the W^T copies): the dgrad reads W_l [out, in] in place as an MN-major B
        # operand (gemm_bf16(b_kn=True)), so no W^T copy exists: one 64 MB transpose pass per 4096 x 4096 layer and step less.
        self.dgrad_kn = (os.environ.get("COLEARN_MLP_DGRAD_KN", "1") == "1") if dgrad_kn is None else bool(dgrad_kn)
        # default (COLEARN_MLP_WGRAD_MN=0: transposed copies): the wgrad reads dz_l [B, out] and a_l [B, in] in place as MN-major
        # operands (gemm_bf16(mn_m=...)): no transposed activations / gradients are written by the producing epilogues
        self.wgrad_mn = (os.environ.get("COLEARN_MLP_WGRAD_MN", "1") == "1") if wgrad_mn is None else bool(wgrad_mn)
        self.dims = list(spec.dims)
        self.L = spec.n_layers
        self.offsets = spec.offsets()
        self.kp = [_pad_to(d) for d in self.dims]          # padded widths
        dev, bf = self.dev, torch.bfloat16
        B = self.B
        self.shadow_arena = shadow                           # bf16 arena written by the two-shot broadcast (or None)
        # bf16 shadows W_l [out_p, in_p] and W_l^T [in_p, out_p]
        self.Ws: List[torch.Tensor] = []
        self.WsT: List[torch.Tensor] = []
        self.exact: List[bool] = []                          # layer needs no padding → fused SGD epilogue allowed
        for l in range(self.L):
            k, n = self.dims[l], self.dims[l + 1]
            exact = (k == self.kp[l] and n == self.kp[l + 1])
            self.exact.append(exact)
            if exact and shadow is not None:
                off = self.offsets[l][0]
                self.Ws.append(shadow[off:off + n * k].view(n, k))   # zero-copy view of the broadcast payload
            else:
                self.Ws.append(torch.zeros(self.kp[l + 1], self.kp[l], device=dev, dtype=bf))
            self.WsT.append(None if self.dgrad_kn else torch.zeros(self.kp[l], self.kp[l + 1], device=dev, dtype=bf))
        self.bias_p = [torch.zeros(self.kp[l + 1], device=dev) for l in range(self.L)]
        # activations (a[0] = padded input) and their transposes, gradients and their transposes
        self.a = [torch.zeros(B, self.kp[l], device=dev, dtype=bf) for l in range(self.L)]
        self.aT = [None if self.wgrad_mn else torch.zeros(self.kp[l], B, device=dev, dtype=bf) for l in range(self.L)]
        self.dz = [torch.zeros(B, self.kp[l + 1], device=dev, dtype=bf) for l in range(self.L)]
        self.dzT = [None if self.wgrad_mn else torch.zeros(self.kp[l + 1], B, device=dev, dtype=bf) for l in range(self.L)]
        self.logits = torch.zeros(B, self.kp[self.L], device=dev)
        self.db = [torch.zeros(self.kp[l + 1], device=dev) for l in range(self.L)]
        # bias-gradient partials written by the dgrad epilogue: one row per 32 batch rows (no atomics)
        self.dbp = [torch.zeros(B // 32, self.kp[l + 1], device=dev) for l in range(self.L)]
        self.dw_edge = {l: torch.zeros(self.kp[l + 1], self.kp[l], device=dev) for l in range(self.L) if not self.exact[l]}
        self.launches = 0
        self._wt_fresh = [False] * self.L                     # W_l^T matches the bf16 shadow W_l

    # -- parameter views -----------------------------------------------------------------------------
    def _w(self, flat: torch.Tensor, l: int) -> torch.Tensor:
        off = self.offsets[l][0]
        return flat[off:off + self.dims[l] * self.dims[l + 1]].view(self.dims[l + 1], self.dims[l])

    def _b(self, flat: torch.Tensor, l: int) -> torch.Tensor:
        off = self.offsets[l][1]
        return flat[off:off + self.dims[l + 1]]

    def chunk_range(self, l: int, chunk_elems: int) -> Tuple[int, int]:
        """[first, last] flag indices covering layer ``l``'s weight + bias in the flat arena."""
        lo = self.offsets[l][0]
        hi = self.offsets[l][1] + self.dims[l + 1] - 1
        return lo // chunk_elems, hi // chunk_elems

    def _refresh_t(self, l: int) -> None:
        """Rebuild ``W_lᵀ`` from the bf16 shadow ``W_l`` (a 64 MB pass for a 4096 × 4096 layer).  The copy is only needed
        by the NEXT dgrad, so the wgrad merely marks it stale and the dgrad refreshes it on demand: the transposes behind
        the last step of a fit — dead work, the next fit starts from ``refresh_exact`` — are never launched."""
        if not self.dgrad_kn:
            ops.transpose_bf16(self.Ws[l], self.WsT[l])
        self._wt_fresh[l] = True

    def sync_transposes(self) -> None:
        """Bring every stale ``W_lᵀ`` up to date (callers that read ``WsT`` outside :meth:`backward`)."""
        for l in range(self.L):
            if not self._wt_fresh[l]:
                self._refresh_t(l)

    def refresh_edge(self, flat: torch.Tensor) -> None:
        """Padded bf16 shadows (+ transposes, padded biases) of the layers that need padding."""
        for l in range(self.L):
            if self.exact[l]:
                continue
            w = self._w(flat, l)
            self.Ws[l].zero_()
            self.Ws[l][: w.shape[0], : w.shape[1]].copy_(w)
            self._refresh_t(l)
            self.bias_p[l].zero_()
            self.bias_p[l][: self.dims[l + 1]].copy_(self._b(flat, l))

    def refresh_exact(self, flat: torch.Tensor, from_broadcast: bool) -> None:
        """bf16 shadow W (skipped when the two-shot broadcast already wrote it) and W^T."""
        for l in range(self.L):
            if not self.exact[l]:
                continue
            if not (from_broadcast and self.shadow_arena is not None):
                self.Ws[l].copy_(ops.fp32_to_bf16(self._w(flat, l).contiguous().view(-1)).view_as(self.Ws[l]))
            self._refresh_t(l)

    def refresh_shadows(self, flat: torch.Tensor, from_broadcast: bool = False) -> None:
        self.refresh_edge(flat)
        self.refresh_exact(flat, from_broadcast)

    def _bias(self, flat: torch.Tensor, l: int) -> torch.Tensor:
        # exact layers read the fp32 master bias straight from the arena (no copy to keep in sync)
        return self._b(flat, l) if self.exact[l] else self.bias_p[l]

    # -- one SGD step = forward() + backward() ------------------------------------------------------------
    def _head_loss(self, z: torch.Tensor, target: torch.Tensor, loss: str):
        """(loss, dL/dz) of the head for ``z[nv, nc]`` (fp32 logits of the valid rows)."""
        if loss == "xent":
            return ops.softmax_xent(z, target.reshape(-1).long())
        y = target.reshape(z.shape).float()
        sig = self.spec.out_activation == "sigmoid"
        if loss == "bce":
            return ops.sigmoid_bce(z, y)                         # fused sigmoid + mean BCE, dz = (p - y) / numel
        out = torch.sigmoid(z) if sig else z
        val, g = ops.sse_loss(out.contiguous(), y, mean=(loss == "mse"))
        return val, (g * out * (1.0 - out) if sig else g)

    def forward(self, flat: torch.Tensor, x: torch.Tensor, labels: torch.Tensor,
                ready: Optional[ReadySpec] = None, loss: str = "xent") -> torch.Tensor:
        """``x``: ``nv <= B`` samples (rows ``nv .. B-1`` of the activations keep whatever finite values they had; their loss
        gradient is zero).  ``ready`` (:class:`ReadySpec`): the GEMMs of the exact layers poll the two-shot broadcast's
        per-chunk flags from their TMA producer warp (first step of a round)."""
        L = self.L
        nv = int(x.shape[0])
        self.a[0][:nv, : self.dims[0]].copy_(x)                  # the padding columns are zero since __init__ and never written
        if not self.wgrad_mn:
            ops.transpose_bf16(self.a[0], self.aT[0])
        for l in range(L):
            kw = {}
            if ready is not None and self.exact[l] and self.shadow_arena is not None:
                kw = dict(ready_flags=ready.flags_ptr, ready_epoch=ready.epoch, ready_chunk_elems=ready.chunk_elems,
                          ready_elem_offset=self.offsets[l][0], ready_epoch_ptr=ready.epoch_ptr)
            if l < L - 1:
                ops.gemm_bf16(self.a[l], self.Ws[l], bias=self._bias(flat, l), relu=True, out_bf16=self.a[l + 1],
                              out_bf16_t=self.aT[l + 1], **kw)
            else:
                ops.gemm_bf16(self.a[l], self.Ws[l], bias=self._bias(flat, l), out_f32=self.logits, **kw)
        nc = self.dims[-1]
        if nv < self._dz_rows:                                   # a shorter batch than before: rows nv.. must carry no gradient
            self.dz[L - 1][nv:self._dz_rows].zero_()
        self._dz_rows = nv
        if loss == "xent" and nc <= 128:
            # one launch: padded fp32 logits -> dL/dz in the padded bf16 GEMM operand, head bias gradient, mean loss
            loss_val = conv_ops.softmax_xent_head(self.logits, labels, nv, nc, dl_bf16=self.dz[L - 1], db=self.db[L - 1])
        else:
            loss_val, dlog = self._head_loss(self.logits[:nv, :nc].contiguous(), labels, loss)
            self.dz[L - 1][:nv, :nc].copy_(dlog)                 # (only the first nc columns are ever written)
            self.db[L - 1][:nc].copy_(dlog.sum(0))
        if not self.wgrad_mn:
            ops.transpose_bf16(self.dz[L - 1], self.dzT[L - 1])
        self.launches += L + 1 + (0 if self.wgrad_mn else 2)       # own kernels: L GEMMs, the loss, two transposes
        return loss_val

    def backward(self, flat: torch.Tensor, lr: float, produced=None) -> None:
        """dgrad with the old weights first, then the (fused) update of layer l.

        ``produced`` (:class:`ops.produced.ProducedSpec`, last step of a round only): fused wgrad → FedAvg reduce.  The
        fused-SGD epilogues report the blocks of final parameters they wrote and everything else that finalises a piece
        of the arena is followed by ``produced.mark`` — every arena element exactly once — so that the overlapped
        two-shot kernel reduces layer ``l`` while layers ``l-1 … 0`` are still in their backward pass.  Wᵀ is not
        rebuilt on that step (the next round derives it from the broadcast)."""
        L = self.L
        end = self.offsets[L - 1][1] + self.dims[L]              # first element after the parameters (arena tail)
        if produced is not None:
            produced.mark(end, produced.n)
        for l in range(L - 1, -1, -1):
            if l > 0:
                if not self._wt_fresh[l]:
                    self._refresh_t(l)
                ops.gemm_bf16(self.dz[l], self.Ws[l] if self.dgrad_kn else self.WsT[l], b_kn=self.dgrad_kn, relu_mask=self.a[l],
                              out_bf16=self.dz[l - 1], out_bf16_t=self.dzT[l - 1], colsum=self.dbp[l - 1],
                              max_ctas=produced.max_ctas if produced is not None else 0)
            if self.exact[l]:
                # fused SGD on the fp32 master + bf16 shadow; W^T is rebuilt by the coalesced transpose kernel
                # (2-byte transposed stores from the epilogue cost more than a separate 64 MB pass)
                self._wgrad(l, sgd_master=self._w(flat, l), sgd_lr=lr, sgd_shadow=self.Ws[l],
                            produced=(produced, self.offsets[l][0]) if produced is not None else None)
                self._wt_fresh[l] = False
            else:
                self._wgrad(l, out_f32=self.dw_edge[l])
                w = self._w(flat, l)
                w.sub_(self.dw_edge[l][: w.shape[0], : w.shape[1]], alpha=lr)
                self.Ws[l][: w.shape[0], : w.shape[1]].copy_(w)
                self._wt_fresh[l] = False
                if produced is not None:
                    produced.mark(self.offsets[l][0], self.offsets[l][0] + w.numel())
            b = self._b(flat, l)
            if l == L - 1:
                b.sub_(self.db[l][: b.shape[0]], alpha=lr)          # head: gradient came from the loss kernel
            else:
                ops.bias_sgd_from_partials(b, self.dbp[l], lr)       # hidden: reduce the epilogue partials + SGD
            if not self.exact[l]:
                self.bias_p[l][: b.shape[0]].copy_(b)
            if produced is not None:
                produced.mark(self.offsets[l][1], self.offsets[l][1] + b.shape[0])
        self.launches += 2 * L + 4

    def _wgrad(self, l: int, **epilogue) -> None:
        """``dW_l = dz_lᵀ · a_l`` with the given epilogue: K-major operands from the transposed copies, or the MN-major form."""
        if self.wgrad_mn:
            ops.gemm_bf16(self.dz[l], self.a[l], mn_m=self.kp[l + 1], **epilogue)
        else:
            ops.gemm_bf16(self.dzT[l], self.aT[l], **epilogue)

    def step(self, flat: torch.Tensor, x: torch.Tensor, labels: torch.Tensor, lr: float, loss: str = "xent") -> torch.Tensor:
        loss_val = self.forward(flat, x, labels, loss=loss)
        self.backward(flat, lr)
        return loss_val

    def n_steps(self, n: int, cfg) -> int:
        """SGD steps of a fit: every epoch walks the whole shard in batches of ``b`` (the last one may be short)."""
        steps = ((n + self.b - 1) // self.b) * cfg.epochs
        if cfg.max_nr_batches and cfg.max_nr_batches > 0:
            steps = min(steps, cfg.max_nr_batches)
        return steps

    def fit(self, flat: torch.Tensor, x: torch.Tensor, y: torch.Tensor, cfg, perm: Optional[torch.Tensor],
            ready: Optional[ReadySpec] = None, wait_chunks=None, produced=None, before_last_backward=None) -> torch.Tensor:
        """Local SGD in place on ``flat`` (full batches only; a tail < batch_size is dropped).

        With ``ready`` (fused broadcast consumption) the order is: wait only for the chunks of the
        padded edge layers → first forward, whose GEMMs poll the per-chunk flags of the big layers
        while the rest of the broadcast is still in flight → ``wait_chunks(None)`` for everything
        (peers must be done reading this rank's arena before SGD writes it) → W^T + backward.

        ``produced`` + ``before_last_backward`` (fused wgrad → FedAvg reduce): the backward of the round's LAST step
        reports what it finalises (:meth:`backward`); the callback runs right before it is queued — the engine launches
        the overlapped two-shot kernel on its side stream there."""
        n, b = x.shape[0], self.b
        total = self.n_steps(n, cfg)
        if ready is not None and wait_chunks is not None:
            for l in range(self.L):
                if not self.exact[l]:
                    wait_chunks(self.chunk_range(l, ready.chunk_elems))
        self.refresh_edge(flat)
        if ready is None:
            self.refresh_exact(flat, from_broadcast=False)
        loss = getattr(cfg, "loss", "xent")
        targets = y.reshape(-1).long() if loss == "xent" else y.reshape(n, -1).float()
        it = 0
        limit = cfg.max_nr_batches if cfg.max_nr_batches and cfg.max_nr_batches > 0 else None
        last = torch.zeros((), device=flat.device)
        for e in range(cfg.epochs):
            order = perm[e % perm.shape[0]].long() if perm is not None else torch.arange(n, device=flat.device)
            for lo in range(0, n, b):                            # the reference's loaders keep the short last batch (C27)
                idx = order[lo:lo + b]
                first = it == 0 and ready is not None
                last = self.forward(flat, x[idx], targets[idx], ready if first else None, loss=loss)
                if first:
                    if wait_chunks is not None:
                        wait_chunks(None)
                    self.refresh_exact(flat, from_broadcast=True)
                final = produced is not None and it == total - 1
                if final and before_last_backward is not None:
                    before_last_backward()
                self.backward(flat, cfg.lr, produced if final else None)
                it += 1
                if limit is not None and it >= limit:
                    return last
        if it == 0 and ready is not None and wait_chunks is not None:
            wait_chunks(None)
        return last

    # -- CUDA graph of a whole local fit (launch-bound inner loop -> one replay per round) -----------------
    def build_round_graph(self, flat: torch.Tensor, x: torch.Tensor, y: torch.Tensor, lr: float, n_steps: int,
                          ready: ReadySpec, n_chunks: int, produced=None) -> None:
        """Capture ``n_steps`` SGD steps of a *fused-broadcast* round into one CUDA graph:

            wait(edge-layer chunks) -> edge shadows -> [gather batch -> forward (GEMMs poll the broadcast
            flags on step 0) -> wait(all chunks) + W^T on step 0 -> backward] x n_steps

        Everything round-specific is device-resident: the epoch the flag waits compare against lives in
        ``ready.epoch_ptr``, the sample order in ``self.g_idx``.  ~45 launches + Python per step collapse
        into one ``replay()``.

        With ``produced`` (fused wgrad → FedAvg reduce) the round is TWO graphs: everything up to the last forward, and
        the last backward with its reports; :meth:`run_round_graph` calls ``between()`` between the two replays (the
        engine launches the overlapped two-shot kernel there, on its side stream)."""
        ext = ops._ext.require()
        dev = flat.device
        self.g_idx = torch.zeros(n_steps, self.B, dtype=torch.long, device=dev)
        self.g_labels = y.reshape(-1).long().contiguous()
        self.g_loss = torch.zeros((), device=dev)
        self.g_steps = n_steps

        def wait(rng):
            if rng is None:
                ext.wait_flags_dev(ready.flags_ptr, n_chunks, ready.epoch_ptr)
            else:
                ext.wait_flags_dev(ready.flags_ptr + 4 * rng[0], rng[1] - rng[0] + 1, ready.epoch_ptr)

        def body():
            for l in range(self.L):
                if not self.exact[l]:
                    wait(self.chunk_range(l, ready.chunk_elems))
            self.refresh_edge(flat)
            loss = None
            for s_i in range(n_steps):
                idx = self.g_idx[s_i]
                loss = self.forward(flat, x.index_select(0, idx), self.g_labels.index_select(0, idx),
                                    ready if s_i == 0 else None)
                if s_i == 0:
                    wait(None)
                    self.refresh_exact(flat, from_broadcast=True)
                if produced is None or s_i < n_steps - 1:
                    self.backward(flat, lr)
            self.g_loss.copy_(loss)

        torch.cuda.synchronize(dev)
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            body()
        self.graph_tail = None
        if produced is not None:
            self.graph_tail = torch.cuda.CUDAGraph()
            with torch.cuda.graph(self.graph_tail):
                self.backward(flat, lr, produced)

    def run_round_graph(self, perm: Optional[torch.Tensor], n: int, between=None) -> torch.Tensor:
        """Replay the captured round on the sample order ``perm`` (int32 ``[epochs, n]`` or None)."""
        need = self.g_steps * self.B
        if perm is None:
            order = torch.arange(need, device=self.g_idx.device) % n
        else:
            flat_perm = perm.reshape(-1)
            if flat_perm.numel() < need:  # several epochs of full batches: drop each epoch's tail like fit()
                per = (n // self.B) * self.B
                flat_perm = perm[:, :per].reshape(-1)
            order = flat_perm[:need]
        self.g_idx.copy_(order.view(self.g_steps, self.B))
        self.graph.replay()
        if getattr(self, "graph_tail", None) is not None:
            if between is not None:
                between()
            self.graph_tail.replay()
        return self.g_loss
