"""Python face of ``mlp_local_sgd_persistent`` (csrc/mlp_persistent.cu) — SURVEY K12.

One launch runs the *entire* local fit of one or many federated clients (one CTA each): the
reference's per-batch ``zero_grad → forward → loss → backward → step`` loop
(``client_federated.py:101-120`` locally; PySyft ``_fit`` remotely, SURVEY C27) never returns to
the host.  Supported architectures are the compile-time instantiations FFNN (10-50-30-10-1,
sigmoid), MLP (10-64-64-2), TestingRemote (2-50-10-1), the autoencoder (10-32-4-32-10, MSE on its input) and the attack-category
FFNN (10-50-30-10-5, softmax cross-entropy); anything else goes through the
layer-wise trainer (``fl/layerwise.py``).
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Optional, Sequence, Tuple, Union

import torch

from . import _ext, host, reference

NET_KINDS = {
    ((10, 50, 30, 10, 1), "sigmoid"): 0,
    ((10, 64, 64, 2), "none"): 1,
    ((2, 50, 10, 1), "none"): 2,
    ((10, 32, 4, 32, 10), "none"): 3,     # the anomaly detector's autoencoder (models/mlp.py AE_SPEC)
    ((10, 50, 30, 10, 5), "none"): 4,     # the attack-category FFNN (models/mlp.py FFNN_CAT_SPEC)
}
NET_FFNN, NET_FFNN_CAT = 0, 4
# Class-weighted fits (csrc/mlp_persistent_cw.cu): net kind -> (classes, losses).  The FFNN's class is its 0 / 1 label, the
# category net's its class index; the weighted instances exist for variant 5 only.
CLASS_WEIGHTED = {NET_FFNN: (2, ("bce", "sse", "mse")), NET_FFNN_CAT: (5, ("xent",))}
CLASS_WEIGHTED_VARIANT = 5
LOSS_CODES = {"bce": 0, "sse": 1, "xent": 2, "mse": 3}
# Kernel variants: 5 = register-resident weights, 128-thread CTA, blocked reduction slices (LDS.128) + pre-scaled dz;
# 6 = 5 with its FMAs written in pairs (Hopper has no packed fp32 FMA: the same FFMA sequence as 5); 3 = strided slices
# (the round-1 default); 1 = smem-resident weights (first version).
# 0 (default) picks variant 5 for every net.
KERNEL_VARIANT = int(__import__("os").environ.get("COLEARN_MLP_VARIANT", "0"))
BEST_VARIANT = {0: 5, 1: 5, 2: 5, 3: 5, 4: 5}    # net kind (NET_KINDS values) -> variant


def resolve_variant(kind: int, variant: Optional[int] = None) -> int:
    v = KERNEL_VARIANT if variant is None else int(variant)
    return BEST_VARIANT.get(kind, 5) if v == 0 else v


PtrLike = Union[torch.Tensor, int, None]


def net_kind_for(dims: Sequence[int], out_activation: str = "none") -> Optional[int]:
    return NET_KINDS.get((tuple(int(d) for d in dims), out_activation))


def _ptr(t: PtrLike) -> int:
    if t is None:
        return 0
    if isinstance(t, torch.Tensor):
        return t.data_ptr()
    return int(t)


@dataclass
class ClientTask:
    """Everything one client CTA needs.  Pointers may be tensors or raw ints (peer memory).

    An empty shard (``x`` with 0 rows, e.g. a trailing virtual client of a short shard) is a valid task: the kernel runs no
    step and reads nothing from ``x``, ``y`` or ``perm``, writes ``out_scale * theta_in`` (0 in delta mode) to ``theta_out``
    and ``{0, 0}`` to ``loss_out``, and still waits on ``wait_flag`` and raises ``signal_flag``."""

    x: torch.Tensor                      # [n, d_in] fp32 CUDA
    y: torch.Tensor                      # [n, y_dim] fp32 CUDA (xent: class index as float)
    theta_in: PtrLike                    # flat arena to start from
    theta_out: PtrLike                   # destination of out_scale * theta_k (or delta)
    perm: Optional[torch.Tensor] = None  # int32 [rows, n]
    loss_out: PtrLike = None             # float[2]: last / mean loss
    wait_flag: PtrLike = None
    wait_value: int = 0
    signal_flag: PtrLike = None
    signal_value: int = 0
    out_scale: float = 1.0
    delta_mode: bool = False
    perm_seed: int = 0                   # != 0 with perm=None: the kernel tabulates the keyed Feistel order itself (before it
    perm_row0: int = 0                   # waits for the broadcast); epoch e = row perm_row0 + e of device_permutation(n, *, perm_seed)
    perm_scratch: Optional[torch.Tensor] = None   # int32 [epochs of the fit * n] device scratch for that table (required with perm_seed)
    _keep: list = field(default_factory=list, repr=False)

    def pack(self) -> bytes:
        ext = _ext.require()
        n = int(self.x.shape[0])
        if self.perm is None and self.perm_seed:
            assert self.perm_scratch is not None and self.perm_scratch.dtype == torch.int32 and self.perm_scratch.numel() >= n, \
                "perm_seed needs an int32 perm_scratch of >= epochs * n elements on the kernel's device"
        y_dim = int(self.y.shape[1]) if self.y.dim() == 2 else 1
        rows = int(self.perm.shape[0]) if self.perm is not None else 1
        return ext.make_client_desc(_ptr(self.x), _ptr(self.y), _ptr(self.perm), _ptr(self.theta_in),
                                    _ptr(self.theta_out), _ptr(self.loss_out), _ptr(self.wait_flag),
                                    int(self.wait_value), _ptr(self.signal_flag), int(self.signal_value),
                                    n, rows, y_dim, float(self.out_scale), int(bool(self.delta_mode)),
                                    int(self.perm_seed) if self.perm is None else 0, int(self.perm_row0), _ptr(self.perm_scratch))


def build_client_descs(tasks: Sequence[ClientTask], device) -> torch.Tensor:
    """Pack descriptors into one uint8 CUDA tensor (pinned staging → async H2D)."""
    blob = b"".join(t.pack() for t in tasks)
    host = torch.frombuffer(bytearray(blob), dtype=torch.uint8)
    if torch.cuda.is_available():
        host = host.pin_memory()
    return host.to(device, non_blocking=True)


def _prep_xy(x: torch.Tensor, y: torch.Tensor, loss: str) -> Tuple[torch.Tensor, torch.Tensor]:
    x = x.contiguous().float()
    y = y.contiguous().float()
    if y.dim() == 1:
        y = y.view(-1, 1)
    return x, y


def check_class_weights(kind: Optional[int], loss: str, class_weights: Sequence[float], variant: Optional[int] = None,
                        cuda: bool = True) -> list:
    """The weights as a list of floats, or ValueError: a class-weighted fit needs a net and loss with weighted instances
    (:data:`CLASS_WEIGHTED`), on CUDA kernel variant 5 (``variant`` / ``COLEARN_MLP_VARIANT``), and one finite weight >= 0 per
    class."""
    if kind not in CLASS_WEIGHTED:
        raise ValueError("class weights: only the FFNN and the attack-category net have class-weighted kernels")
    classes, losses = CLASS_WEIGHTED[kind]
    if loss not in losses:
        raise ValueError(f"class weights: loss {loss!r} not supported for this net (use {', '.join(losses)})")
    if cuda and resolve_variant(kind, variant) != CLASS_WEIGHTED_VARIANT:
        raise ValueError(f"class weights: only kernel variant {CLASS_WEIGHTED_VARIANT} has class-weighted instances, "
                         f"not {resolve_variant(kind, variant)}")
    w = [float(v) for v in class_weights]
    if len(w) != classes:
        raise ValueError(f"class weights: {len(w)} values for {classes} classes")
    for c, v in enumerate(w):
        if not (math.isfinite(v) and v >= 0.0):
            raise ValueError(f"class weights: weight {v!r} of class {c} is not a finite number >= 0")
    return w


def check_local_opt(local_opt, class_weights=None):
    """The optimizer to launch on the optimizer instances (``csrc/mlp_persistent_opt.cu``), or None for plain SGD (``None`` or
    a plain ``LocalOpt``: the kernels of before optimizers existed).  ValueError for anything but a ``fl.local_opt.LocalOpt``
    and for class weights next to an optimizer (the weighted instances are variant 5's, the optimizer instances variant 1's)."""
    from ..fl.local_opt import LocalOpt
    if local_opt is None:
        return None
    if not isinstance(local_opt, LocalOpt):
        raise ValueError(f"local_opt must be a fl.local_opt.LocalOpt, got {type(local_opt).__name__}")
    if local_opt.is_plain():
        return None
    if class_weights is not None:
        raise ValueError("class weights together with a local optimizer are not supported")
    return local_opt


def mlp_local_sgd_multi(dims: Sequence[int], out_activation: str, descs: torch.Tensor, n_clients: int,
                        batch_size: int = 1, lr: float = 0.01, epochs: int = 1, max_nr_batches: int = -1,
                        loss: str = "xent", desc_offset: int = 0, variant: Optional[int] = None,
                        class_weights: Optional[Sequence[float]] = None, local_opt=None) -> None:
    """Launch ``n_clients`` CTAs from a packed descriptor tensor (see :func:`build_client_descs`).

    The labels behind the descriptors are not checked here (they are device memory the caller packed).  For the
    attack-category net they must be class indices in [0, 5): the kernel stays memory-safe for any other value (its heads
    select z_y by compare-and-select or ``label & 31``), but trains on a wrong gradient.  Every data path that feeds this
    (the CSV adapter, ``synthetic_category``) validates its codes when it loads them; :func:`mlp_local_sgd` checks them.  The
    same holds for the 0 / 1 labels of a class-weighted FFNN fit.

    ``class_weights``: a class-weighted fit (``reference.loss_and_dz``), launched on the weighted instances; the weights, net,
    loss and variant are checked before the launch (:func:`check_class_weights`).

    ``local_opt``: a ``fl.local_opt.LocalOpt``.  None or plain SGD launches what it always launched; any other optimizer
    launches the optimizer instances (variant 1's shared-memory kernel with the ``local_opt.cuh`` step), whatever ``variant``
    says."""
    kind = net_kind_for(dims, out_activation)
    if kind is None:
        raise ValueError(f"no persistent-kernel instantiation for dims={tuple(dims)} act={out_activation}")
    if loss == "bce" and out_activation != "sigmoid":
        raise ValueError("bce needs a sigmoid head")
    lo = check_local_opt(local_opt, class_weights)
    if lo is not None:
        _ext.require().mlp_local_sgd_opt(kind, descs, int(desc_offset), int(n_clients), int(batch_size), int(epochs),
                                         int(max_nr_batches if max_nr_batches is not None else -1), LOSS_CODES[loss], float(lr),
                                         lo.launch_args())
        return
    args = (kind, descs, int(desc_offset), int(n_clients), int(batch_size), int(epochs),
            int(max_nr_batches if max_nr_batches is not None else -1), LOSS_CODES[loss], float(lr), resolve_variant(kind, variant))
    if class_weights is None:
        _ext.require().mlp_local_sgd(*args)
    else:
        w = check_class_weights(kind, loss, class_weights, variant)
        _ext.require().mlp_local_sgd_cw(*args, w)


def mlp_local_sgd(flat: torch.Tensor, dims: Sequence[int], x: torch.Tensor, y: torch.Tensor,
                  perm: Optional[torch.Tensor], batch_size: int = 1, lr: float = 0.01, epochs: int = 1,
                  max_nr_batches: int = -1, loss: str = "xent", out_activation: str = "none",
                  return_mean: bool = False, variant: Optional[int] = None,
                  class_weights: Optional[Sequence[float]] = None, local_opt=None) -> torch.Tensor:
    """Single-client in-place local SGD on ``flat``; returns the last batch loss (0-dim tensor).

    CPU tensors run ``reference.mlp_local_sgd`` (identical semantics); CUDA tensors run the
    persistent kernel — there is no silent fallback on CUDA.  The attack-category net refuses, before any launch, a label that
    is not a class index in [0, 5): the kernel's head selects z_y by that index.

    ``class_weights``: a class-weighted fit (FFNN: 2 weights, for labels 0 and 1; attack-category net: 5), refused before any
    launch unless :func:`check_class_weights` accepts it and every label is a class index.

    ``local_opt``: the fit's ``fl.local_opt.LocalOpt`` (see :func:`mlp_local_sgd_multi`); on CPU the host executor's generic
    loop or ``reference.mlp_local_sgd`` takes its step."""
    local_opt = check_local_opt(local_opt, class_weights)
    kind = net_kind_for(dims, out_activation)
    if class_weights is not None:
        class_weights = check_class_weights(kind, loss, class_weights, variant, cuda=flat.is_cuda)
        check_class_labels(y, len(class_weights))
    elif kind == NET_FFNN_CAT:
        check_class_labels(y, int(dims[-1]))
    if not flat.is_cuda:
        # CPU devices: the native host executor (csrc/mlp_host.cpp) when it is built and the arena can be trained in
        # place, else the PyTorch definitions (identical semantics; the executor is tested against them)
        if (host.available() and flat.dtype == torch.float32 and flat.is_contiguous() and not flat.requires_grad
                and out_activation in ("none", "sigmoid")):
            res = host.mlp_local_sgd_multi(dims, out_activation, [flat], [x], [y], [perm], batch_size, lr, epochs,
                                           max_nr_batches, loss, threads=1, class_weights=class_weights, local_opt=local_opt)
            return res[0, 1 if return_mean else 0].clone()
        if perm is None:
            perm = reference.make_permutation(x.shape[0], epochs, 0, shuffle=False)
        cw = None if class_weights is None else torch.tensor(class_weights, dtype=torch.float32).to(flat.dtype)
        return reference.mlp_local_sgd(flat, dims, x, y, perm, batch_size, lr, epochs, max_nr_batches, loss, out_activation, cw,
                                       local_opt)
    x, y = _prep_xy(x, y, loss)
    loss_out = torch.zeros(2, device=flat.device, dtype=torch.float32)
    if perm is not None:
        perm = perm.to(flat.device, torch.int32).contiguous()
    task = ClientTask(x=x, y=y, theta_in=flat, theta_out=flat, perm=perm, loss_out=loss_out)
    descs = build_client_descs([task], flat.device)
    mlp_local_sgd_multi(dims, out_activation, descs, 1, batch_size, lr, epochs, max_nr_batches, loss, variant=variant,
                        class_weights=class_weights, local_opt=local_opt)
    return loss_out[1 if return_mean else 0]


def check_class_labels(y: torch.Tensor, classes: int) -> None:
    """ValueError unless every label is an integer class index in [0, classes)"""
    v = y.detach().reshape(-1).double()
    bad = ~((v == v.floor()) & (v >= 0) & (v < classes))
    if bool(bad.any()):
        i = int(bad.nonzero()[0, 0])
        raise ValueError(f"label {float(v[i])!r} of row {i} is not a class index in [0, {classes})")


def mlp_forward(flat: torch.Tensor, dims: Sequence[int], x: torch.Tensor, out_activation: str = "none") -> torch.Tensor:
    """Batched forward of a small MLP from its flat arena (inference / evaluation)."""
    if not flat.is_cuda:
        return reference.mlp_forward(flat, dims, x, out_activation)[0]
    kind = net_kind_for(dims, out_activation)
    if kind is None:
        raise ValueError(f"no persistent-kernel instantiation for dims={tuple(dims)}")
    return _ext.require().mlp_forward(kind, flat.contiguous(), x.contiguous().float(), int(dims[-1]))
