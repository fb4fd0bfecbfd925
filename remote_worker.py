#!/usr/bin/env python
"""CoLearn device-side worker CLI (flag-compatible with the reference ``remote_worker.py:18-47``).

    python remote_worker.py --host 127.0.0.1 -p 8778 -b localhost -t "topic/state" -w 1 \
        -e "TRAINING" --verbose -dt <training csv> -di <inference csv>

The host MUST be given as an IP (it is what the coordinator parses out of the event).  The worker
hosts its dataset under key ``"training"`` (rw.py:108), optional inference tensors tagged
``"inference"`` (rw.py:102-104), an optional held-out set under ``"evaluation"`` (``-de`` / ``--eval-fraction``) for
federated evaluation, announces itself on the bus after ``--wait`` seconds
(rw.py:110-114) and then serves fit/search/predict RPCs forever (rw.py:117).
"""
import argparse
import logging
import os
import sys
from threading import Timer

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


# (flags, kwargs): the nine reference options first (same spellings and defaults), then the extensions
_OPTIONS = (
    (("--port", "-p"), dict(type=int, default=8777, help="TCP port the worker's RPC server listens on")),
    (("--host",), dict(type=str, required=True, help="IPv4 address of this device (it is what the coordinator parses out of the event)")),
    (("--broker", "-b"), dict(type=str, required=True, help="MQTT broker to announce to")),
    (("--topic", "-t"), dict(type=str, required=True, help="topic the coordinator listens on")),
    (("--wait", "-w"), dict(type=float, default=5, help="delay in seconds between start-up and the announcement")),
    (("--event", "-e"), dict(type=str, default="TRAINING", help="what to announce: TRAINING, INFERENCE or NOT_READY")),
    (("--training", "-dt"), dict(type=str, default=None, help="Bot-IoT CSV hosted as the private training set")),
    (("--inference", "-di"), dict(type=str, default=None, help="Bot-IoT CSV whose rows are hosted as inference tensors")),
    (("--verbose", "-v"), dict(action="store_true", help="log every RPC")),
    (("--evaluation", "-de"), dict(type=str, default=None, help="CSV hosted as the held-out set the coordinator's federated "
                                                                 "evaluation scores the global model on (only counts leave the device)")),
    (("--eval-fraction",), dict(type=float, default=0.0, help="hold this fraction of the training rows out as the evaluation set "
                                                              "(a seeded random subset, see fl/fedeval.py split_eval), in (0, 1)")),
    (("--broker-port",), dict(type=int, default=1883)),
    (("--synthetic",), dict(type=int, default=0, help="host N synthetic rows instead of --training")),
    (("--data-model",), dict(default="ffnn", help="architecture the synthetic data is shaped for (resnet18: 32x32 images, net: "
                                                  "28x28, testing_remote: 2 features, ffnn_category: five attack categories, "
                                                  "otherwise the ten UNSW-IoT features)")),
    (("--seed",), dict(type=int, default=0)),
    (("--dataset",), dict(default="unsw", help="dataset adapter that reads -dt / -di (data.register_dataset; default: the Bot-IoT CSV adapter)")),
    (("--plugin",), dict(action="append", default=[], metavar="MODULE_OR_FILE",
                         help="import this module / .py file first: it may call models.register_model / data.register_dataset (repeatable)")),
    (("--no-cuda",), dict(action="store_true", help="serve fits on the CPU even if a GPU is present")),
    (("--no-will",), dict(action="store_true", help="do not register the NOT_READY last-will with the broker")),
    (("--broker-wait",), dict(type=float, default=30.0, metavar="SECONDS",
                              help="keep retrying for this long when the broker is not reachable yet (devices often boot before it)")),
    (("--reannounce",), dict(type=float, default=0.0, metavar="SECONDS",
                             help="repeat the announcement every SECONDS (the coordinator deregisters a device after each training; "
                                  "the reference's devices have to publish again by hand). 0 = announce once, like the reference")),
    (("--tls-ca",), dict(default=None, help="CA bundle: verify the broker; with --tls-cert also demand a client certificate from the coordinator")),
    (("--tls-cert",), dict(default=None, help="this device's certificate (RPC server side and client certificate towards the broker)")),
    (("--tls-key",), dict(default=None, help="private key belonging to --tls-cert")),
    (("--tls-no-verify-hostname",), dict(action="store_true", help="verify the broker's certificate chain only, not its name / IP SAN")),
)


def build_parser() -> argparse.ArgumentParser:
    parser = argparse.ArgumentParser(description="CoLearn device: hosts a private dataset and serves fit / search / predict RPCs.")
    for flags, kwargs in _OPTIONS:
        parser.add_argument(*flags, **kwargs)
    return parser


def pick_dataset(args):
    """--synthetic N > the CSV given with -dt > the reference's XOR toy set (rw.py:75-80).  Synthetic rows made for an
    attack-category model (--data-model ffnn_category) keep their class indices as the dataset's categories, next to the
    binary attack label, like a Bot-IoT CSV."""
    from colearn_federated_learning_b200.data import load_dataset, xor_toy_dataset
    from colearn_federated_learning_b200.fl import targets

    if args.synthetic > 0:
        return targets.synthetic_dataset(args.data_model, args.synthetic, seed=args.seed)
    if args.training:
        logging.info("training data: %s", args.training)
        return load_dataset(args.dataset, args.training)
    return xor_toy_dataset()


def main(args: argparse.Namespace) -> None:  # pragma: no cover - exercised by the CLI integration tests
    import torch

    from colearn_federated_learning_b200.control.bus import BusClient
    from colearn_federated_learning_b200.control.event_parser import format_event
    from colearn_federated_learning_b200.control.workers import WorkerServer
    from colearn_federated_learning_b200.data import load_dataset
    from colearn_federated_learning_b200.models import load_plugins

    load_plugins(args.plugin)
    logging.basicConfig(format="%(asctime)s: %(message)s", level=logging.INFO, datefmt="%H:%M:%S")
    identity = f"{args.host}:{args.port}"
    on_gpu = torch.cuda.is_available() and not args.no_cuda
    from colearn_federated_learning_b200.control.tls import contexts_from_cli
    rpc_tls = contexts_from_cli(args.tls_ca, args.tls_cert, args.tls_key, server=True,
                                require_client_cert=bool(args.tls_ca)) if args.tls_cert else None   # rw.py:60-61
    server = WorkerServer(identity, args.host, args.port, device=torch.device("cuda" if on_gpu else "cpu"), verbose=args.verbose,
                          ssl_context=rpc_tls)
    server.add_dataset(pick_dataset(args), key="training")                       # rw.py:108
    if args.evaluation and args.eval_fraction > 0:
        raise SystemExit("-de and --eval-fraction both define the evaluation set: give one of them")
    if args.evaluation:
        logging.info("evaluation data: %s", args.evaluation)
        server.add_dataset(load_dataset(args.dataset, args.evaluation), key="evaluation")
    elif args.eval_fraction > 0:
        server.hold_out_evaluation(args.eval_fraction, args.seed)
    if args.inference:
        logging.info("inference data: %s", args.inference)
        rows = load_dataset(args.dataset, args.inference).data
        server.load_data([torch.as_tensor(r).float() for r in rows], tag="inference")   # rw.py:102-104

    # one bus identity per device (the reference's shared literal id gets duplicates kicked, SURVEY §2.8-12)
    bus = BusClient(client_id="worker-" + identity, transport="tcp")
    bus_tls = contexts_from_cli(args.tls_ca, args.tls_cert, args.tls_key, server=False,
                                check_hostname=not args.tls_no_verify_hostname)
    if bus_tls is not None:
        bus.tls_set(context=bus_tls)
    if not args.no_will:
        # if this process dies without a DISCONNECT the broker withdraws the device on our behalf
        bus.will_set(args.topic, format_event(args.host, "NOT_READY", args.port))
    import time
    deadline = time.monotonic() + max(0.0, args.broker_wait)
    while True:
        try:
            bus.connect(args.broker, args.broker_port)
            break
        except OSError as e:                                                      # refused / unreachable: the broker may still be starting
            if time.monotonic() >= deadline:
                raise
            logging.info("broker %s:%d not reachable yet (%r), retrying", args.broker, args.broker_port, e)
            time.sleep(0.5)
    announcement = format_event(args.host, args.event, args.port)
    def announce() -> None:
        bus.publish(args.topic, announcement)
        if args.reannounce > 0:                                                   # stay available for the next windows
            again = Timer(args.reannounce, announce)
            again.daemon = True
            again.start()

    delayed = Timer(args.wait, announce)                                          # rw.py:110-114
    delayed.daemon = True
    delayed.start()
    try:
        server.start()                                                            # serve forever (rw.py:117)
    except KeyboardInterrupt:
        server.stop()
        bus.disconnect()


if __name__ == "__main__":
    main(build_parser().parse_args())
