"""colearn_federated_learning_b200 — a Hopper (sm_90a) native federated-averaging engine.

Capabilities mirror CoLearn (aferaudo/CoLearn_Federated_Learning): publish/subscribe device
admission (TRAINING / INFERENCE / NOT_READY), temporal-window worker collection, multi-round
FedAvg over private shards, IoT allow-list, on-worker inference, ``.pth`` checkpoints, and an
SMPC training demo — redesigned so that coordinator/worker roles map onto the GPUs of one
NVSwitch box and every hot path is a hand-written CUDA kernel.

Layer map (see DESIGN.md):
    control/   event grammar, registry, pub/sub bus, temporal window, selection, coordinator
    fl/        FedAvg, local/remote/encrypted trainers, evaluate, inference
    models/    FFNN, TestingRemote, Net, MLP, WideMLP, ResNet-18 + flat-arena specs
    data/      NetworkTrafficDataset, transforms, federate(), synthetic UNSW generator
    ops/       sm_90a kernels (persistent MLP local-SGD, wgmma GEMMs, losses, SGD, ...)
    parallel/  symmetric memory arena, fused broadcast / FedAvg-reduce kernels, round engine
    smpc/      fixed-point additive secret sharing (SPDZ-style) for the encrypted demo
    utils/     checkpoint, metrics, monitors, timing
"""

__version__ = "0.1.0"

from . import settings  # noqa: F401  (reference-compatible global registry)
