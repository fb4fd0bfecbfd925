#!/usr/bin/env python
"""CoLearn coordinator CLI (flag-compatible with the reference ``federated_coordinator.py:64-90``).

    python federated_coordinator.py -t "topic/state"          # local (VirtualWorker) case
    python federated_coordinator.py -t "topic/state" -r       # remote case

Events are published to the bus as ``"(192.168.1.7, TRAINING)"`` (local) or
``"(127.0.0.1, 8777, TRAINING)"`` (remote) — e.g. with ``python -m
colearn_federated_learning_b200.tools.bus_pub -t topic/state -m "(192.168.1.7, TRAINING)"``, the
stand-in for ``mosquitto_pub``.  ``--host embedded`` (default when ``--host localhost`` has no
broker listening) starts the TCP bus broker inside this process.

On a multi-GPU box launch it under torchrun with ``--box``: rank 0 hosts the coordinator role,
every rank is a worker, and the broadcast / FedAvg legs run as fused NVLink kernels
(``colearn_federated_learning_b200.parallel``).
"""
import argparse
import logging
import os
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from colearn_federated_learning_b200.control.arguments import Arguments  # noqa: E402
from colearn_federated_learning_b200.models import MODEL_REGISTRY  # noqa: E402


def build_parser() -> argparse.ArgumentParser:
    parser = argparse.ArgumentParser(description="Run Federated coordinator")
    # --- reference flags (fc.py:64-90) ---------------------------------------------------------
    parser.add_argument("--port", "-p", type=int, default=1883, help="port number of the where the broker is listining (default 1883)")
    parser.add_argument("--host", type=str, default="localhost", help="broker ip address (default localhost)")
    parser.add_argument("--topic", "-t", type=str, required=True, help="topic where the event must be published")
    parser.add_argument("--remote", "-r", action="store_true", help="Remote learning activation")
    parser.add_argument("--window", "-w", type=int, default=1, help="temporal window size (default 1)")
    parser.add_argument("--encryption", "-e", action="store_true", help="Simulates the encryption on two virtual workes")
    parser.add_argument("--federated_round", "-f", type=int, default=1, help="number of federated rounds (round > 1 trains 1000 batches per round)")
    parser.add_argument("--iot", "-i", action="store_true", help="enable iot validation (IP allow-list)")
    # --- everything the reference hard-codes in Arguments / Coordinator.__init__ ------------------
    d = Arguments()
    parser.add_argument("--model", choices=sorted(MODEL_REGISTRY), default=d.model)
    parser.add_argument("--loss", default=d.loss, choices=["auto", "bce", "sse", "xent", "mse"])
    parser.add_argument("--batch-size", type=int, default=d.batch_size)
    parser.add_argument("--local-epochs", type=int, default=d.epochs)
    parser.add_argument("--max-batches", type=int, default=d.federate_after_n_batches, help="local SGD steps per round (-1 = full epoch; rounds>1 default to 1000)")
    parser.add_argument("--lr", type=float, default=d.lr)
    parser.add_argument("--server-lr", type=float, default=None,
                        help="server learning rate (default: 1.0 for --server-opt sgd / avgm, 0.01 for adagrad / adam / yogi)")
    parser.add_argument("--server-opt", choices=["sgd", "avgm", "adagrad", "adam", "yogi"], default=d.server_opt,
                        help="server optimizer on top of the FedAvg average: sgd = plain FedAvg, avgm = server momentum, "
                             "adagrad / adam / yogi = adaptive (Reddi et al. 2021); its state is not checkpointed")
    parser.add_argument("--server-beta1", type=float, default=d.server_beta1, help="first-moment decay of --server-opt, in [0, 1)")
    parser.add_argument("--server-beta2", type=float, default=d.server_beta2, help="second-moment decay of adam / yogi, in [0, 1)")
    parser.add_argument("--server-tau", type=float, default=d.server_tau, help="adaptivity of adagrad / adam / yogi (> 0)")
    parser.add_argument("--aggregator", choices=["mean", "median", "trimmed_mean", "geomed", "norm_clip"], default=d.aggregator,
                        help="how the client models are combined: mean = (weighted) FedAvg; median / trimmed_mean = coordinate-wise, "
                             "unweighted, robust to a minority of bad clients (not with --weighted); geomed = weighted geometric "
                             "median (RFA), norm_clip = weighted mean of the updates clipped to --clip-norm: distance-based, "
                             "take --weighted (local and remote mode; not with --uplink-codec topk or --secure-agg)")
    parser.add_argument("--trim-fraction", type=float, default=d.trim_fraction,
                        help="trimmed_mean: fraction of the values dropped at each end of every parameter, in [0, 0.5)")
    parser.add_argument("--geomed-iters", type=int, default=d.geomed_iters,
                        help="geomed: smoothed Weiszfeld steps from the current model, in 1..16 (each one more read of the replies)")
    parser.add_argument("--geomed-eps", type=float, default=d.geomed_eps,
                        help="geomed: floor nu of the distances in the weights alpha_k / max(nu, d_k), finite and > 0")
    parser.add_argument("--clip-norm", type=float, default=None,
                        help="norm_clip (required with it): L2 bound tau of every device's update; a device moves the model by at "
                             "most alpha_k tau")
    parser.add_argument("--uplink-codec", choices=["fp32", "int8", "int4", "topk"], default=d.uplink,
                        help="what a device sends back after a fit: fp32 = its model; int8 / int4 = its delta to the received model, "
                             "stochastically quantized with one scale per 256 parameters (~3.9x / ~7.5x fewer bytes); topk = the "
                             "--uplink-topk largest entries of every 256 of its delta plus what it did not send before (error "
                             "feedback; ~25x fewer bytes at 8); local and remote mode only (not with --box or -e)")
    parser.add_argument("--uplink-topk", type=int, default=d.uplink_topk,
                        help="--uplink-codec topk: entries sent per block of 256 parameters, in 1..32 (not with a robust --aggregator)")
    parser.add_argument("--downlink-codec", choices=["fp32", "int8", "int4", "topk"], default=d.downlink,
                        help="what the coordinator sends after the first round of a training: fp32 = the model; int8 / int4 / topk = "
                             "the same codecs as --uplink-codec applied to the model minus the replica every device keeps, one "
                             "encode per round for all devices (needs --uplink-codec int8, int4 or topk; not with --box or -e)")
    parser.add_argument("--downlink-topk", type=int, default=d.downlink_topk,
                        help="--downlink-codec topk: entries sent per block of 256 parameters, in 1..32")
    parser.add_argument("--secure-agg", action="store_true",
                        help="remote mode: secure aggregation (Bonawitz et al. 2017): every device sends its delta as pairwise-masked "
                             "fixed-point words, the coordinator learns only their sum; devices that drop out before replying are "
                             "tolerated (not with --uplink-codec, a robust --aggregator, --weighted, --box, -e or local mode)")
    parser.add_argument("--secagg-clip", type=float, default=d.secagg_clip,
                        help="--secure-agg: every coordinate of a device's delta is clipped to [-C, C] before the fixed-point code (finite, > 0)")
    parser.add_argument("--seed", type=int, default=d.seed)
    parser.add_argument("--log-interval", type=int, default=d.log_interval)
    parser.add_argument("--test-path", type=str, default=d.test_path, help="CSV used by local/encrypted mode and evaluation")
    parser.add_argument("--synthetic", type=int, default=0, help="use N synthetic UNSW-shaped rows instead of --test-path")
    parser.add_argument("--dataset", default="unsw", help="dataset adapter that reads --test-path (data.register_dataset; default: the Bot-IoT CSV adapter)")
    parser.add_argument("--plugin", action="append", default=[], metavar="MODULE_OR_FILE",
                        help="import this module / .py file first: it may call models.register_model / data.register_dataset "
                             "(the reference's 'use your own model/dataset' without editing sources; repeatable)")
    parser.add_argument("--weighted", action="store_true", help="sample-count weighted FedAvg (default: uniform, like the reference)")
    parser.add_argument("--select", type=int, default=None, help="train at most k of the collected workers")
    parser.add_argument("--selection", choices=["all", "first", "random"], default="all")
    parser.add_argument("--checkpoint", type=str, default="./test.pth")
    parser.add_argument("--save-every", type=int, default=0, help="also write the checkpoint every N rounds (0 = only after the last round, like the reference)")
    parser.add_argument("--dtype", choices=["fp32", "bf16"], default=d.dtype,
                        help="--box: bf16 makes the FedAvg broadcast carry a bf16 copy of the model next to the fp32 master "
                             "(consumed directly by the wgmma GEMMs of the wide / conv models)")
    parser.add_argument("--no-cuda", action="store_true")
    parser.add_argument("--strict-events", action="store_true", help="validate IPv4 octets / full match (reference is lax)")
    parser.add_argument("--fit-timeout", type=float, default=None, help="seconds before a silent remote worker is dropped from a round")
    parser.add_argument("--filter-file", type=str, default=None)
    parser.add_argument("--metrics", type=str, default=None, help="write per-round JSONL here")
    parser.add_argument("--round-log", type=str, default=None, help="write the reference-format round log here")
    parser.add_argument("--metrics-port", type=int, default=0, help="serve Prometheus metrics (rounds, round time, losses, traffic) on this port")
    parser.add_argument("--evaluate", action="store_true", help="evaluate the global model on --test-path after training")
    parser.add_argument("--fed-eval-every", type=int, default=d.fed_eval_every, metavar="N",
                        help="federated evaluation: after every N-th round and after the last one the devices score the global model on "
                             "rows they keep out of training and return counts; the round record gets fed_eval (detection rate, "
                             "false-alarm rate, precision, F1, ROC-AUC, average precision). 0 = off")
    parser.add_argument("--eval-bins", type=int, default=d.eval_bins, help="--fed-eval-every: score histogram bins (power of two, 2..4096)")
    parser.add_argument("--eval-threshold", type=float, default=d.eval_threshold,
                        help="--fed-eval-every: a one-column model flags a row as an attack iff its score is above this")
    parser.add_argument("--eval-fraction", type=float, default=d.eval_fraction,
                        help="--fed-eval-every in local and box mode: fraction of every device's shard held out for evaluation, in (0, 1) "
                             "(remote devices hold theirs out themselves: remote_worker.py -de / --eval-fraction)")
    parser.add_argument("--alarm-fpr", type=float, default=d.alarm_fpr,
                        help="--model autoencoder: the federated alarm threshold is the lowest error bin at which at most this fraction "
                             "of the devices' held-out benign rows raise an alarm, in (0, 1)")
    parser.add_argument("--async-buffer", type=int, default=d.async_buffer, metavar="K",
                        help="remote mode: asynchronous buffered aggregation (FedBuff): devices train whenever they are free, from the "
                             "current global version, and the server steps once K replies are buffered, each weighted by (1 + "
                             "staleness)^-a; -f then counts server steps. 0 = synchronous rounds (not with --secure-agg, a compressed "
                             "--downlink-codec, --box, -e, local mode or models with BatchNorm buffers)")
    parser.add_argument("--async-concurrency", type=int, default=d.async_concurrency, metavar="C",
                        help="--async-buffer: fits in flight at once (0 = one per selected device)")
    parser.add_argument("--max-staleness", type=int, default=d.max_staleness, metavar="S",
                        help="--async-buffer: a reply trained from a model more than S versions old is dropped")
    parser.add_argument("--staleness-exponent", type=float, default=d.staleness_exponent, metavar="A",
                        help="--async-buffer: a reply of staleness tau weighs (1 + tau)^-A (0.5 = FedBuff's 1/sqrt(1 + tau))")
    parser.add_argument("--embedded-broker", action="store_true", help="start the TCP bus broker inside this process")
    parser.add_argument("--tls-ca", default=None, help="CA bundle: verify the broker / the devices (and, with --tls-cert on the embedded broker, demand client certificates)")
    parser.add_argument("--tls-cert", default=None, help="certificate for the embedded broker / client certificate towards broker and devices")
    parser.add_argument("--tls-key", default=None, help="private key belonging to --tls-cert")
    parser.add_argument("--tls-no-verify-hostname", action="store_true",
                        help="verify the certificate chain only, not that the certificate names the broker / device address")
    parser.add_argument("--inject", action="append", default=[], metavar="SPEC",
                        help="fault injection on the embedded broker: drop:<regex> | dup:<regex> | delay:<seconds>:<regex> (repeatable)")
    parser.add_argument("--exit-after", type=int, default=0, help="exit after N completed trainings (0 = run forever)")
    parser.add_argument("--box", action="store_true", help="multi-GPU box mode under torchrun (rank 0 = coordinator)")
    parser.add_argument("--backend", choices=["auto", "fused", "nccl", "cpu"], default="auto")
    parser.add_argument("--clients-per-gpu", type=int, default=1, help="--box: virtual federated devices hosted by each GPU (one CTA each)")
    parser.add_argument("--enc-items", type=int, default=None, help="-e: number of samples that are secret-shared and trained on (reference: 1000)")
    parser.add_argument("--round-deadline-ms", type=float, default=0.0,
                        help="--box: a selected worker that has not delivered its model this many ms after the coordinator started its "
                             "reduce is dropped from that round (weights renormalised); 0 = wait for everyone")
    parser.add_argument("--box-event", default="TRAINING", help="--box: the state every rank announces at start (rw.py --event)")
    parser.add_argument("--box-script", default=None, metavar="RANK:STATE:AFTER[,...]",
                        help="--box: further events, e.g. '3:NOT_READY:0,2:INFERENCE:1' = rank 3 withdraws right after its announcement, "
                             "rank 2 asks for inference once it has seen one training complete")
    parser.add_argument("--box-no-reannounce", action="store_true",
                        help="--box: devices do not ask for training again after a training they took part in")
    parser.add_argument("--box-inference-rows", type=int, default=5, help="--box: rows of its shard every rank tags as inference data")
    return parser


def arguments_from_cli(ns: argparse.Namespace) -> Arguments:
    a = Arguments()
    a.model, a.loss, a.batch_size, a.epochs = ns.model, ns.loss, ns.batch_size, ns.local_epochs
    a.federate_after_n_batches, a.lr, a.seed = ns.max_batches, ns.lr, ns.seed
    from colearn_federated_learning_b200.fl.server_opt import default_server_lr
    a.server_opt = getattr(ns, "server_opt", "sgd")
    a.server_lr = ns.server_lr if ns.server_lr is not None else default_server_lr(a.server_opt)
    a.server_beta1 = getattr(ns, "server_beta1", a.server_beta1)
    a.server_beta2 = getattr(ns, "server_beta2", a.server_beta2)
    a.server_tau = getattr(ns, "server_tau", a.server_tau)
    a.server_optimizer()              # rejects a beta outside [0, 1) / tau <= 0 before anything starts
    a.log_interval, a.test_path, a.synthetic, a.weighted = ns.log_interval, ns.test_path, ns.synthetic, ns.weighted
    a.aggregator = getattr(ns, "aggregator", a.aggregator)
    a.trim_fraction = getattr(ns, "trim_fraction", a.trim_fraction)
    a.geomed_iters = getattr(ns, "geomed_iters", a.geomed_iters)
    a.geomed_eps = getattr(ns, "geomed_eps", a.geomed_eps)
    clip_norm = getattr(ns, "clip_norm", None)
    a.clip_norm = a.clip_norm if clip_norm is None else clip_norm
    a.client_aggregator()             # rejects a trim fraction outside [0, 0.5) and --weighted with a robust kind
    a.uplink = getattr(ns, "uplink_codec", a.uplink)
    a.uplink_topk = getattr(ns, "uplink_topk", a.uplink_topk)
    a.uplink_codec()                  # rejects a topk k outside 1..32 and topk with a robust aggregator
    a.downlink = getattr(ns, "downlink_codec", a.downlink)
    a.downlink_topk = getattr(ns, "downlink_topk", a.downlink_topk)
    a.secure_agg = bool(getattr(ns, "secure_agg", False))
    a.secagg_clip = getattr(ns, "secagg_clip", a.secagg_clip)
    a.secagg_clip_value()             # rejects a bad clip and --secure-agg with an uplink codec, a robust aggregator or --weighted
    a.downlink_codec()                # rejects a topk k outside 1..32 and a compressed downlink with an fp32 uplink
    a.no_cuda, a.backend = ns.no_cuda, ns.backend
    if getattr(ns, "enc_items", None):
        a.n_train_items_enc = int(ns.enc_items)
    a.dtype, a.save_every = ns.dtype, max(0, ns.save_every)
    a.dataset = ns.dataset
    a.fed_eval_every = getattr(ns, "fed_eval_every", a.fed_eval_every)
    a.eval_bins = getattr(ns, "eval_bins", a.eval_bins)
    a.eval_threshold = getattr(ns, "eval_threshold", a.eval_threshold)
    a.eval_fraction = getattr(ns, "eval_fraction", a.eval_fraction)
    a.alarm_fpr = getattr(ns, "alarm_fpr", a.alarm_fpr)
    a.fed_eval_settings()             # rejects bins / threshold / fraction outside their ranges and --secure-agg with it
    a.async_buffer = getattr(ns, "async_buffer", a.async_buffer)
    a.async_concurrency = getattr(ns, "async_concurrency", a.async_concurrency)
    a.max_staleness = getattr(ns, "max_staleness", a.max_staleness)
    a.staleness_exponent = getattr(ns, "staleness_exponent", a.staleness_exponent)
    a.async_settings()                # rejects negative settings and --async-buffer with --secure-agg or a compressed downlink
    return a


def main(args: argparse.Namespace) -> None:
    logging.basicConfig(format="%(asctime)s: %(message)s", level=logging.INFO, datefmt="%H:%M:%S")
    logging.info(os.getpid())
    if args.box:
        from colearn_federated_learning_b200.parallel.box import run_box_coordinator
        run_box_coordinator(args, arguments_from_cli(args))
        return

    from colearn_federated_learning_b200.control.bus import TcpBroker
    from colearn_federated_learning_b200.control.coordinator import Coordinator
    from colearn_federated_learning_b200.utils.metrics import RoundLogger
    import socket
    import time

    from colearn_federated_learning_b200.control.tls import contexts_from_cli

    broker = None
    client_tls = contexts_from_cli(args.tls_ca, args.tls_cert, args.tls_key, server=False,
                                   check_hostname=not args.tls_no_verify_hostname)
    if args.embedded_broker:
        server_tls = contexts_from_cli(args.tls_ca, args.tls_cert, args.tls_key, server=True,
                                       require_client_cert=bool(args.tls_ca)) if args.tls_cert else None
        broker = TcpBroker("127.0.0.1" if args.host == "localhost" else args.host, args.port, ssl_context=server_tls).start()
        logging.info("embedded bus broker listening on %s:%d", broker.host, broker.port)
        for spec in args.inject:
            broker.broker.inject_from_spec(spec)
            logging.info("fault injection active: %s", spec)
    exporter = None
    if args.metrics_port:
        from colearn_federated_learning_b200.utils.metrics import PrometheusExporter
        exporter = PrometheusExporter(args.metrics_port)
        logging.info("Prometheus metrics on http://127.0.0.1:%d/metrics", exporter.port)
    coordinator = Coordinator(args.window, args.remote, args.federated_round, args.encryption, args.iot,
                              args=arguments_from_cli(args), transport="tcp", path=args.checkpoint,
                              strict_events=args.strict_events, select_k=args.select, selection=args.selection,
                              fit_timeout=args.fit_timeout, filter_file=args.filter_file,
                              metrics=RoundLogger(args.metrics, args.round_log, exporter=exporter), evaluate_after=args.evaluate,
                              worker_ssl_context=client_tls)
    if client_tls is not None:
        coordinator.tls_set(context=client_tls)
    try:
        if args.exit_after > 0:
            coordinator.run(args.host, args.port, args.topic, forever=False)
            # a window whose training raised counts too (it is in the scheduler's history with an "error" entry):
            # otherwise one failing training would keep this loop spinning forever
            def finished() -> int:
                failed = sum(1 for rec in coordinator.windower.history if "error" in rec)
                return coordinator.trainings_done + failed
            while finished() < args.exit_after:
                time.sleep(0.05)
            if coordinator.windower.last_error is not None:
                logging.error("last training failed: %r", coordinator.windower.last_error)
            coordinator.shutdown()
        else:
            coordinator.run(args.host, args.port, args.topic)
    except (ConnectionRefusedError, socket.gaierror) as e:
        logging.error("cannot reach the bus broker at %s:%d (%r); start one with --embedded-broker", args.host, args.port, e)
        sys.exit(2)
    finally:
        if broker is not None:
            broker.stop()


def parse_cli(argv=None) -> argparse.Namespace:
    """Plugins are imported before the real parser is built, so that ``--model`` accepts what they register."""
    pre = argparse.ArgumentParser(add_help=False)
    pre.add_argument("--plugin", action="append", default=[])
    known, _ = pre.parse_known_args(argv)
    if known.plugin:
        from colearn_federated_learning_b200.models import load_plugins
        load_plugins(known.plugin)
    parser = build_parser()
    ns = parser.parse_args(argv)
    try:
        arguments_from_cli(ns)           # the server optimizer and aggregator settings (beta in [0, 1), tau > 0, trim in [0, 0.5))
    except ValueError as e:
        parser.error(str(e))
    if ns.uplink_codec != "fp32" and (ns.box or ns.encryption):
        parser.error(f"--uplink-codec {ns.uplink_codec} applies to the local and remote modes only: --box trains on the GPUs of one "
                     "box (fp32 models over NVLink) and -e exchanges secret shares")
    if ns.downlink_codec != "fp32" and (ns.box or ns.encryption):
        parser.error(f"--downlink-codec {ns.downlink_codec} applies to the local and remote modes only: --box broadcasts fp32 models "
                     "over NVLink and -e exchanges secret shares")
    if ns.aggregator in ("geomed", "norm_clip") and (ns.box or ns.encryption):
        parser.error(f"--aggregator {ns.aggregator} applies to the local and remote modes only: --box reduces the models across the "
                     "GPUs in one pass (no per-step distances) and -e exchanges secret shares")
    if ns.fed_eval_every > 0:
        if ns.encryption:
            parser.error("--fed-eval-every applies to the local, remote and box modes: -e exchanges secret shares")
        if not ns.remote and not ns.eval_fraction > 0:
            parser.error("--fed-eval-every in local and box mode needs --eval-fraction > 0: the rows every device holds out")
        if ns.remote and ns.eval_fraction > 0:
            parser.error("--eval-fraction applies to local and box mode: remote devices hold their evaluation rows out themselves "
                         "(remote_worker.py -de / --eval-fraction)")
        from colearn_federated_learning_b200.fl.fedeval import check_model
        from colearn_federated_learning_b200.models import build_model
        try:
            check_model(build_model(ns.model))
        except ValueError as e:
            parser.error(f"--fed-eval-every with --model {ns.model}: {e}")
    from colearn_federated_learning_b200.fl import anomaly
    if anomaly.is_autoencoder(MODEL_REGISTRY.get(ns.model)):
        try:
            anomaly.check_settings(ns, box=ns.box, encryption=ns.encryption)
        except ValueError as e:
            parser.error(str(e))
    from colearn_federated_learning_b200.fl import category
    if category.is_category(MODEL_REGISTRY.get(ns.model)):
        if ns.box:
            parser.error(f"--model {ns.model} does not run in box mode (--box): box mode trains on the binary attack label")
        if ns.encryption:
            parser.error(f"--model {ns.model} does not run with -e: the secret-shared training takes the binary attack label")
    if ns.secure_agg:
        if ns.box or ns.encryption or not ns.remote:
            parser.error("--secure-agg applies to remote mode (-r) only: in local mode every update is in the coordinator's process "
                         "anyway, --box trains on the GPUs of one box and -e exchanges secret shares")
        from colearn_federated_learning_b200.models import build_model
        if any(b.is_floating_point() for b in build_model(ns.model).buffers()):
            parser.error(f"--secure-agg does not apply to --model {ns.model}: its floating-point buffers (BatchNorm running "
                         "statistics) would travel in the clear")
    if ns.async_buffer:
        if ns.box or ns.encryption or not ns.remote:
            parser.error("--async-buffer applies to remote mode (-r) only: local mode and --box train their workers in lockstep "
                         "launches and -e exchanges secret shares")
        from colearn_federated_learning_b200.models import build_model
        if any(b.is_floating_point() for b in build_model(ns.model).buffers()):
            parser.error(f"--async-buffer does not apply to --model {ns.model}: averaging its BatchNorm statistics across model "
                         "versions is not defined")
    return ns


if __name__ == "__main__":
    main(parse_cli())
