"""Put the UNMODIFIED reference under ``oracle/_ref`` (git-ignored), for the reference arm of ``bench.py`` and its tests.

The reference is a flat tree of scripts without ``setup.py`` / ``pyproject.toml``, meant to be run from its checkout, so
``pip install --target`` cannot install it; the "install" is a byte-identical copy of the Python sources + the example
dataset + the allow-list, with a ``SHA256SUMS`` manifest that ``verify()`` re-checks before every reference-arm run.
Nothing here imports the product package.  ``__graft_entry__.build()`` calls :func:`install_if_available`.

    python oracle/install_ref.py [--src <reference checkout>]

The checkout is ``--src``, else ``$COLEARN_REFERENCE_SRC``, else ``/root/reference``.
"""
from __future__ import annotations

import hashlib
import os
import shutil
import sys
from typing import Dict

HERE = os.path.dirname(os.path.abspath(__file__))
DEST = os.path.join(HERE, "_ref")
DEFAULT_SRC = os.environ.get("COLEARN_REFERENCE_SRC", "/root/reference")
FILES = ["federated_coordinator.py", "client_federated.py", "remote_worker.py", "datasets.py", "event_parser.py", "settings.py",
         "README.md", "device_filtering/filtering_file.txt", "device_filtering/file_upgrader.py",
         "dataset_example/UNSW_2018_IoT_Botnet_Final_10_best_Training_1_1.csv"]


def _sha(path: str) -> str:
    h = hashlib.sha256()
    with open(path, "rb") as f:
        h.update(f.read())
    return h.hexdigest()


def install(src: str = DEFAULT_SRC, dest: str = DEST) -> Dict[str, str]:
    sums = {}
    for rel in FILES:
        s, d = os.path.join(src, rel), os.path.join(dest, rel)
        if not os.path.exists(s):
            continue
        os.makedirs(os.path.dirname(d), exist_ok=True)
        shutil.copyfile(s, d)
        sums[rel] = _sha(d)
        assert sums[rel] == _sha(s)
    with open(os.path.join(dest, "SHA256SUMS"), "w") as f:
        for rel, h in sorted(sums.items()):
            f.write(f"{h}  {rel}\n")
    return sums


def verify(dest: str = DEST) -> Dict[str, str]:
    """Re-hash the installed files against the manifest written at install time; returns {file: sha256}."""
    manifest = os.path.join(dest, "SHA256SUMS")
    if not os.path.exists(manifest):
        raise FileNotFoundError(f"{manifest} missing: run `python oracle/install_ref.py --src <reference checkout>`")
    sums = {}
    with open(manifest) as f:
        for line in f:
            h, rel = line.strip().split("  ", 1)
            if _sha(os.path.join(dest, rel)) != h:
                raise RuntimeError(f"oracle/_ref/{rel} differs from the installed reference file")
            sums[rel] = h
    return sums


def install_if_available(src: str = DEFAULT_SRC) -> bool:
    """Install from ``src`` when it is a reference checkout; leave ``oracle/_ref`` as it is otherwise.  True if installed."""
    if not os.path.exists(os.path.join(src, "federated_coordinator.py")):
        return False
    install(src)
    return True


if __name__ == "__main__":
    src = sys.argv[sys.argv.index("--src") + 1] if "--src" in sys.argv else DEFAULT_SRC
    for rel, h in sorted(install(src).items()):
        print(h, rel)
