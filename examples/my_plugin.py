"""Example plugin: "use your own model / dataset" (the reference's README.md:119-169) without editing any source.

    # coordinator (local VirtualWorker mode on the CSV below)
    python federated_coordinator.py -t topic/state --embedded-broker --plugin examples/my_plugin.py \
        --model tiny_mlp --dataset two_moons_csv --test-path /tmp/moons.csv
    # device
    python remote_worker.py --host 127.0.0.1 -p 8777 -b 127.0.0.1 -t topic/state --plugin examples/my_plugin.py \
        --dataset two_moons_csv -dt /tmp/moons.csv

Both sides load the same plugin: models travel as flat parameter vectors (never as code), so a worker must know the
architecture it is asked to train by name.
"""
import csv

import torch

from colearn_federated_learning_b200.data import BaseDataset, register_dataset
from colearn_federated_learning_b200.models import MLPNet, MLPSpec, register_model


class TinyMLP(MLPNet):
    """2-16-16-2 classifier.  Any ``MLPNet`` trains through the native executors (persistent kernel instantiations,
    layer-wise wgmma trainer, CPU host executor); other ``nn.Module``s use the autograd path."""

    def __init__(self) -> None:
        super().__init__(MLPSpec((2, 16, 16, 2), "none", "xent"))


def two_moons_csv(path: str) -> BaseDataset:
    """CSV with rows ``x0,x1,label`` -> ``BaseDataset(data [N, 2], targets [N, 1])``."""
    rows = [[float(v) for v in r] for r in csv.reader(open(path)) if r and not r[0].startswith("#")]
    t = torch.tensor(rows, dtype=torch.float32)
    return BaseDataset(t[:, :2].contiguous(), t[:, 2:3].contiguous())


register_model("tiny_mlp", TinyMLP, default_loss="xent", overwrite=True)
register_dataset("two_moons_csv", two_moons_csv, overwrite=True)
