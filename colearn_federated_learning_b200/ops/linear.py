"""wgmma GEMM front-end (csrc/gemm_wgmma.cu) — SURVEY K7/K8.

``C[M,N] = A[M,K] · B[N,K]^T`` with both operands K-major bf16, fp32 accumulation in registers and a
fused epilogue (bias / ReLU / ReLU-mask / fp32+bf16+transposed outputs / fused SGD / bias-grad
column sums / fused broadcast-consumption flags).  Shapes must satisfy ``M%128 == N%128 == 0``
and ``K%64 == 0``; callers pad (see ``fl/layerwise.py``).  CPU tensors use the fp32 reference.
"""
from __future__ import annotations

from typing import Optional

import torch

from . import _ext


def gemm_bf16(a: torch.Tensor, b: torch.Tensor, *, bias: Optional[torch.Tensor] = None, relu: bool = False,
              relu_mask: Optional[torch.Tensor] = None, out_bf16: Optional[torch.Tensor] = None,
              out_f32: Optional[torch.Tensor] = None, out_bf16_t: Optional[torch.Tensor] = None,
              sgd_master: Optional[torch.Tensor] = None, sgd_lr: float = 0.0,
              sgd_shadow: Optional[torch.Tensor] = None, sgd_shadow_t: Optional[torch.Tensor] = None,
              colsum: Optional[torch.Tensor] = None, ready_flags: int = 0, ready_epoch: int = 0,
              ready_chunk_elems: int = 1, ready_elem_offset: int = 0, tile_n: int = 0,
              ready_epoch_ptr: int = 0, cluster: int = 0, split_k: int = 0,
              split_out: Optional[torch.Tensor] = None, mn_m: int = 0, b_kn: bool = False,
              addend: Optional[torch.Tensor] = None, produced=None, max_ctas: int = 0) -> None:
    """Launch the wgmma GEMM; results land in the provided output tensors.

    ``mn_m = M > 0`` selects the "MN-major" form ``C[M, N] = Aᵀ·B`` for ``a[K, a_cols]`` (``a_cols <= M``, the missing
    columns count as zeros) and ``b[K, N]``, both row-major: the reduction runs over *rows*, which is how the conv
    wgrad ``dW[Cout, k] = Σ_pixels dz[pixel, Cout]·col[pixel, k]`` finds its operands in memory (no transposes).
    ``b_kn=True`` keeps ``a[M, K]`` K-major and takes ``b[rows >= K, N]`` row-major (``C = A·B[:K]``) — the conv dgrad
    against the packed weights ``Wp[Cout, K]``, so no ``Wᵀ`` copy is needed.

    ``addend`` (bf16 ``[M, N]``) is added to the accumulator before the bf16 / fp32 outputs are written (the residual
    gradient joining a dgrad).

    ``split_k = S > 1`` (skinny problems: few output tiles, long reduction): the K range is cut into S slices that
    run as independent work units; slice ``s`` stores its raw fp32 accumulator to ``split_out[s]`` (``[S, M, N]``)
    and no other epilogue option may be given — ``ops.conv.splitk_reduce`` sums the slices and applies the epilogue.

    ``produced = (ProducedSpec, elem_offset)`` (with ``sgd_master``, a view of the work arena starting at element
    ``elem_offset``): fused wgrad → FedAvg reduce — each epilogue warp reports the block of final parameters it wrote
    (``ops.produced``), and ``ProducedSpec.max_ctas`` caps the persistent grid so that the overlapped two-shot kernel
    keeps its SMs; ``max_ctas`` alone caps the grid of a GEMM that only runs next to that kernel (the dgrads of the
    last backward)."""
    prod_arg = [0, 0, int(max_ctas)] if max_ctas else []
    if produced is not None:
        assert sgd_master is not None and not (split_k and split_k > 1), "produced reports come from the fused-SGD epilogue"
        if produced[0].sig is not None:
            prod_arg = produced[0].gemm_arg(produced[1])
    from . import conv as _conv
    # tests (ops.conv.simt()): CPU bf16 operands go to the kernel SOURCE on the functional wgmma / TMA / mbarrier model
    simt_mod = (_conv._EMUL["mod"] if (not a.is_cuda and _conv._EMUL["on"] and hasattr(_conv._EMUL["mod"], "gemm_tcgen05")
                                       and a.dtype == torch.bfloat16 and not ready_flags and not cluster) else None)
    if mn_m:
        assert a.shape[0] == b.shape[0] and a.shape[1] <= mn_m and mn_m % 128 == 0 and a.shape[1] % 8 == 0
        assert not ready_flags and not cluster, "the MN-major form has no cluster / ready-flag variant"
        if not a.is_cuda and simt_mod is None:   # reference: bring the operands to the K-major form of the definition below
            at = a.new_zeros(mn_m, a.shape[0])
            at[: a.shape[1]].copy_(a.t())
            a, b, mn_m = at, b.t().contiguous(), 0
    if b_kn:
        assert not mn_m and a.shape[1] <= b.shape[0] and not ready_flags and not cluster
        if not a.is_cuda and simt_mod is None:
            b, b_kn = b[: a.shape[1]].t().contiguous(), False
    m_out, n_out = (mn_m, b.shape[1]) if mn_m else (a.shape[0], b.shape[1] if b_kn else b.shape[0])
    k_red = a.shape[0] if mn_m else a.shape[1]
    if split_k and split_k > 1:
        assert split_out is not None and split_out.numel() >= split_k * m_out * n_out
        assert (bias is None and not relu and relu_mask is None and out_bf16 is None and out_f32 is None and out_bf16_t is None
                and sgd_master is None and colsum is None and not ready_flags and addend is None), "split-K stores raw partials only"
        assert k_red // 64 >= split_k, "split_k must not exceed K/64"
    if simt_mod is not None:
        simt_mod.gemm_tcgen05(a.contiguous(), b.contiguous(), bias, bool(relu), relu_mask, out_bf16, out_f32, out_bf16_t, sgd_master,
                              float(sgd_lr), sgd_shadow, sgd_shadow_t, colsum, int(tile_n), int(split_k or 0), split_out, int(mn_m or 0),
                              bool(b_kn), addend, [], prod_arg)
        return
    if not a.is_cuda:
        if split_k and split_k > 1:   # same slice boundaries as the kernel: k-blocks of 64, slice s = [nkb*s/S, nkb*(s+1)/S)
            nkb = a.shape[1] // 64
            part = split_out[: split_k * a.shape[0] * b.shape[0]].view(split_k, a.shape[0], b.shape[0])
            for s_ in range(split_k):
                lo, hi = nkb * s_ // split_k * 64, nkb * (s_ + 1) // split_k * 64
                part[s_].copy_(a[:, lo:hi].float() @ b[:, lo:hi].float().t())
            return
        acc = a.float() @ b.float().t()
        if bias is not None:
            acc = acc + bias
        if relu:
            acc = torch.relu(acc)
        if relu_mask is not None:
            acc = acc * (relu_mask.float() > 0)
        if addend is not None:
            acc = acc + addend.float()
        if colsum is not None:   # [M/32, N] per-32-row-block partial column sums
            colsum.copy_(acc.view(acc.shape[0] // 32, 32, acc.shape[1]).sum(1))
        if sgd_master is not None:
            sgd_master.sub_(sgd_lr * acc)
            if sgd_shadow is not None:
                sgd_shadow.copy_(sgd_master)
            if sgd_shadow_t is not None:
                sgd_shadow_t.copy_(sgd_master.t())
            if produced is not None:
                produced[0].mark(produced[1], produced[1] + sgd_master.numel())
            return
        if out_f32 is not None:
            out_f32.copy_(acc)
        if out_bf16 is not None:
            out_bf16.copy_(acc)
        if out_bf16_t is not None:
            out_bf16_t.copy_(acc.t())
        return
    _ext.require().gemm_tcgen05(a, b, bias, bool(relu), relu_mask, out_bf16, out_f32, out_bf16_t, sgd_master,
                                float(sgd_lr), sgd_shadow, sgd_shadow_t, colsum, int(ready_flags), int(ready_epoch),
                                int(ready_chunk_elems), int(ready_elem_offset), int(tile_n), int(ready_epoch_ptr), int(cluster),
                                int(split_k or 0), split_out, int(mn_m or 0), bool(b_kn), addend, [], prod_arg)


def linear_forward(x: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor] = None, relu: bool = False,
                   out_dtype: torch.dtype = torch.bfloat16) -> torch.Tensor:
    """``relu?(x @ w.T + bias)`` for bf16 ``x[M,K]``, ``w[N,K]`` (tile-aligned shapes)."""
    m, n = x.shape[0], w.shape[0]
    out = torch.empty(m, n, device=x.device, dtype=out_dtype)
    if out_dtype == torch.bfloat16:
        gemm_bf16(x, w, bias=bias, relu=relu, out_bf16=out)
    else:
        gemm_bf16(x, w, bias=bias, relu=relu, out_f32=out)
    return out


def transpose_bf16(x: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """``out[C,R] = x[R,C]^T`` for bf16 (smem-tiled kernel on CUDA)."""
    if not x.is_cuda:
        res = x.t().contiguous()
        if out is not None:
            out.copy_(res)
            return out
        return res
    return _ext.require().transpose_bf16(x.contiguous(), out)


def bias_sgd_from_partials(bias: Optional[torch.Tensor], partials: torch.Tensor, lr: float) -> torch.Tensor:
    """``bias[:] -= lr * partials.sum(0)[:len(bias)]`` (partials = the GEMM epilogue's bias-gradient partial
    sums); returns the summed gradient."""
    if not partials.is_cuda:
        g = partials.sum(0)
        if bias is not None:
            bias.sub_(g[: bias.numel()], alpha=lr)
        return g
    return _ext.require().bias_sgd_from_partials(bias, partials.contiguous(), float(lr))
