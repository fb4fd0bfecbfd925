"""Hyper-parameter object.

Parity: reference ``Arguments`` (``federated_coordinator.py:45-61``): batch_size 1,
test_batch_size 1024, epochs 1, federate_after_n_batches -1 (unlimited), lr 0.01, momentum 0.5
(unused by the reference's plain SGD), seed 1, log_interval 30, test_path = example CSV; setter
``set_federated_batches``.  Everything the reference hard-codes is a field here and is exposed
as a CLI flag by ``federated_coordinator.py`` with the reference value as default.
"""
from __future__ import annotations

from dataclasses import dataclass, asdict
from typing import Any, Dict, Optional, Tuple

DEFAULT_TEST_PATH = "./dataset_example/UNSW_2018_IoT_Botnet_Final_10_best_Training_1_1.csv"
ROUND_MODE_BATCHES = 1000  # reference: ``round > 1`` forces 1000 local batches (fc.py:533-535)


@dataclass
class Arguments:
    batch_size: int = 1
    test_batch_size: int = 1024
    epochs: int = 1
    federate_after_n_batches: int = -1
    lr: float = 0.01
    momentum: float = 0.5
    no_cuda: bool = False
    seed: int = 1
    log_interval: int = 30
    save_model: bool = False
    test_path: str = DEFAULT_TEST_PATH
    # -- extensions (not in the reference) -------------------------------------------------
    model: str = "ffnn"
    loss: str = "auto"             # auto | bce | sse | xent
    weighted: bool = False         # False = uniform FedAvg (reference), True = n_k / sum(n)
    server_lr: float = 1.0         # theta <- theta + server_lr * avg_delta (1.0 = plain FedAvg)
    server_opt: str = "sgd"        # server optimizer: sgd (plain FedAvg) | avgm | adagrad | adam | yogi (fl/server_opt.py);
                                   # the CLI's --server-lr defaults to 0.01 for the adaptive kinds, 1.0 otherwise
    server_beta1: float = 0.9
    server_beta2: float = 0.99
    server_tau: float = 1e-3
    aggregator: str = "mean"       # mean (weighted FedAvg) | median | trimmed_mean (coordinate-wise, unweighted) | geomed | norm_clip
                                   # (distance-based, weighted; fl/aggregate.py)
    trim_fraction: float = 0.1     # trimmed_mean: fraction of the values dropped at each end, in [0, 0.5)
    geomed_iters: int = 3          # geomed: smoothed Weiszfeld steps, in 1..16
    geomed_eps: float = 1e-6       # geomed: distance floor nu of the weights alpha_k / max(nu, d_k), finite and > 0
    clip_norm: float = 0.0         # norm_clip: L2 bound tau of every update (finite, > 0; required with norm_clip)
    uplink: str = "fp32"           # what a device sends back after a fit: fp32 (its model) | int8 | int4 (its quantized delta) |
                                   # topk (the largest entries of its delta, with error feedback; fl/uplink.py)
    uplink_topk: int = 8           # topk: entries kept per block of 256 parameters, in 1..32
    downlink: str = "fp32"         # what the coordinator sends after round 0: fp32 (the model) | int8 | int4 | topk (a compressed
                                   # delta to the replica the devices keep; needs a delta uplink; fl/uplink.py)
    downlink_topk: int = 8         # downlink topk: entries sent per block of 256 parameters, in 1..32
    secure_agg: bool = False       # remote mode: devices send pairwise-masked fixed-point deltas, the coordinator learns only their
                                   # sum (fl/secagg.py)
    secagg_clip: float = 1.0       # secure aggregation: every coordinate of a delta is clipped to [-clip, clip] (finite, > 0)
    fed_eval_every: int = 0        # >0: the devices score the global model on held-out rows after every N-th round and the last one
                                   # (fl/fedeval.py); 0: no federated evaluation
    eval_bins: int = 256           # federated evaluation: score histogram bins, a power of two in [2, 4096]
    eval_threshold: float = 0.5    # federated evaluation: a one-column model predicts the positive class iff p > threshold
    eval_fraction: float = 0.0     # federated evaluation, local and box mode: fraction of every device's shard held out, in (0, 1)
    alarm_fpr: float = 0.01        # autoencoder: the alarm threshold lets at most this fraction of the held-out benign rows raise an
                                   # alarm, in (0, 1) (fl/anomaly.py)
    class_weight: Optional[str] = None   # class-weighted local fits (fl/classweight.py): "balanced" (from the federated class
                                   # counts) or C comma-separated weights; None: unweighted
    class_weight_max: float = 10.0  # balanced class weights: the cap of every weight (> 0)
    local_optimizer: str = "SGD"   # the devices' local optimizer (fl/local_opt.py): "SGD" or "Adam"
    local_momentum: float = 0.0    # SGD momentum in [0, 1) (not `momentum` above: the reference's 0.5 there was never applied)
    local_nesterov: bool = False   # SGD: nesterov momentum
    local_weight_decay: float = 0.0  # SGD / Adam: L2 weight decay (>= 0)
    local_betas: Tuple[float, float] = (0.9, 0.999)  # Adam: (beta1, beta2), each in [0, 1)
    local_eps: float = 1e-8        # Adam: eps (> 0)
    async_buffer: int = 0          # remote mode: >0 = asynchronous buffered aggregation, one server step per K replies from devices
                                   # that train from whatever version is current (fl/asyncagg.py); 0 = synchronous rounds
    async_concurrency: int = 0     # asynchronous: fits in flight (0 = one per selected device)
    max_staleness: int = 4         # asynchronous: replies trained from a model more than S versions old are dropped
    staleness_exponent: float = 0.5  # asynchronous: a reply of staleness tau weighs (1 + tau)^-a
    backend: str = "auto"          # auto | fused | nccl | cpu
    dtype: str = "fp32"            # fp32 | bf16 (box mode: bf16 shadow of the broadcast for the wgmma consumers)
    save_every: int = 0            # >0: checkpoint every N rounds, not only after the last one
    synthetic: int = 0             # >0: generate this many synthetic UNSW-shaped rows
    dataset: str = "unsw"          # data.DATASET_REGISTRY entry that reads test_path (user datasets: data.register_dataset)
    n_train_items_enc: int = 1000  # fc.py:432
    precision_fractional: int = 3  # fc.py:433

    def local_opt(self):
        """The :class:`fl.local_opt.LocalOpt` of every device's fit.  ValueError for settings out of range, and for a setting of
        the other optimizer (momentum or nesterov with Adam, betas or eps with SGD) rather than ignoring it."""
        from ..fl.local_opt import LocalOpt
        other = {"SGD": ("local_betas", "local_eps"), "Adam": ("local_momentum", "local_nesterov")}.get(self.local_optimizer, ())
        default = Arguments()
        for name in other:
            if getattr(self, name) != getattr(default, name):
                flag = "--" + name.replace("_", "-")
                raise ValueError(f"{flag} does not apply to --local-optimizer {self.local_optimizer}")
        if self.local_optimizer == "SGD":
            return LocalOpt("SGD", momentum=self.local_momentum, nesterov=self.local_nesterov, weight_decay=self.local_weight_decay)
        return LocalOpt(self.local_optimizer, weight_decay=self.local_weight_decay, betas=tuple(self.local_betas), eps=self.local_eps)

    def server_optimizer(self):
        """The :class:`fl.server_opt.ServerOpt` these arguments describe (``server_lr`` is its learning rate)."""
        from ..fl.server_opt import ServerOpt
        return ServerOpt(self.server_opt, lr=self.server_lr, beta1=self.server_beta1, beta2=self.server_beta2, tau=self.server_tau)

    def client_aggregator(self):
        """The :class:`fl.aggregate.Aggregator` these arguments describe; a coordinate-wise kind refuses ``weighted`` (it is
        unweighted), the distance-based kinds take it."""
        from ..fl.aggregate import Aggregator
        clip = self.clip_norm if self.aggregator == "norm_clip" else None
        agg = Aggregator(self.aggregator, self.trim_fraction, iters=self.geomed_iters, eps=self.geomed_eps, clip_norm=clip)
        if agg.coordinate_wise and self.weighted:
            raise ValueError(f"--weighted does not apply to aggregator {self.aggregator!r}: the median / trimmed mean are unweighted")
        return agg

    def uplink_codec(self):
        """The :class:`fl.uplink.UplinkCodec` of the devices' replies; topk refuses a robust aggregator (a coordinate-wise
        median of sparse deltas is 0 wherever fewer than half the devices sent that coordinate)."""
        from ..fl.uplink import UplinkCodec
        codec = UplinkCodec(self.uplink, k=self.uplink_topk)
        agg = self.client_aggregator()
        if codec.sparse and agg.coordinate_wise:
            raise ValueError(f"--uplink-codec topk does not combine with --aggregator {self.aggregator}: only the mean of sparse deltas keeps the update")
        if codec.sparse and agg.distance_based:
            raise ValueError(f"--uplink-codec topk does not combine with --aggregator {self.aggregator}: the distances of sparse "
                             "deltas would measure which entries the codec kept, not how far a device moved")
        return codec

    def downlink_codec(self):
        """The :class:`fl.uplink.UplinkCodec` of the model sent to the devices; a compressed one needs a delta uplink (int8 /
        int4 / topk): the devices' deltas are then taken against the replica they trained from."""
        from ..fl.uplink import UplinkCodec
        codec = UplinkCodec(self.downlink, k=self.downlink_topk)
        if codec.kind != "fp32" and self.uplink_codec().kind == "fp32" and not self.secure_agg:
            raise ValueError(f"--downlink-codec {self.downlink} needs --uplink-codec int8, int4 or topk: with fp32 replies the server "
                             "would have to shift every returned model by theta - replica")
        return codec

    def secagg_clip_value(self) -> float:
        """The clip of ``secure_agg`` after the checks that do not depend on the mode: the devices send fixed-point deltas
        whose sum the coordinator learns, so there is no other uplink codec, no robust aggregator and no weighting."""
        from ..fl.secagg import check_clip
        clip = check_clip(self.secagg_clip)
        if not self.secure_agg:
            return clip
        if self.uplink != "fp32":
            raise ValueError(f"--secure-agg does not combine with --uplink-codec {self.uplink}: the masked row is its own encoding")
        agg = self.client_aggregator()
        if agg.coordinate_wise:
            raise ValueError(f"--secure-agg does not combine with --aggregator {self.aggregator}: only the sum of the updates survives the masks")
        if agg.distance_based:
            raise ValueError(f"--secure-agg does not combine with --aggregator {self.aggregator}: the per-device distances it weighs by "
                             "are hidden by the masks")
        if self.weighted:
            raise ValueError("--secure-agg does not combine with --weighted: the masked sum gives the unweighted mean")
        return clip

    def fed_eval_settings(self) -> None:
        """The checks of the federated-evaluation settings that do not depend on the mode (ValueError with the reason)."""
        if self.fed_eval_every < 0:
            raise ValueError(f"--fed-eval-every must be >= 0, not {self.fed_eval_every}")
        if self.eval_bins < 2 or self.eval_bins > 4096 or self.eval_bins & (self.eval_bins - 1):
            raise ValueError(f"--eval-bins must be a power of two in [2, 4096], not {self.eval_bins}")
        if not 0.0 <= self.eval_threshold <= 1.0:
            raise ValueError(f"--eval-threshold must be in [0, 1], not {self.eval_threshold}")
        if not 0.0 <= self.eval_fraction < 1.0:
            raise ValueError(f"--eval-fraction must be in [0, 1), not {self.eval_fraction}")
        if not 0.0 < self.alarm_fpr < 1.0:
            raise ValueError(f"--alarm-fpr must be in (0, 1), not {self.alarm_fpr}")
        if self.eval_fraction > 0 and self.fed_eval_every == 0:
            raise ValueError("--eval-fraction holds rows out for --fed-eval-every, which is not set")
        if self.fed_eval_every > 0 and self.secure_agg:
            raise ValueError("--fed-eval-every does not combine with --secure-agg: every device's counts (and with them the label mix "
                             "of its data, which secure aggregation hides) would travel in the clear")

    def async_settings(self):
        """The :class:`fl.asyncagg.AsyncSettings` of the ``async_*`` fields, None for synchronous rounds; refuses the settings it
        cannot run with whatever the mode: secure aggregation (its masks cancel only over a synchronous cohort) and a compressed
        downlink (one coordinator replica is only valid when every device has seen every broadcast)."""
        from ..fl.asyncagg import optional_settings
        st = optional_settings(self.async_buffer, self.async_concurrency, self.max_staleness, self.staleness_exponent)
        if st is not None and self.secure_agg:
            raise ValueError("--async-buffer does not combine with --secure-agg: the pairwise masks cancel only over a synchronous cohort")
        if st is not None and self.downlink != "fp32":
            raise ValueError(f"--async-buffer does not combine with --downlink-codec {self.downlink}: the coordinator's one replica is "
                             "only valid when every device has seen every broadcast")
        return st

    def set_federated_batches(self, batches: int) -> None:
        self.federate_after_n_batches = batches

    def to_dict(self) -> Dict[str, Any]:
        return asdict(self)
