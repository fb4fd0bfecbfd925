#!/usr/bin/env python
"""Process / NIC monitor kept at the reference's path (``data/ps_util_test.py``): ``-p <pid>`` and/or ``-n <iface>``;
``--gpu <index>`` additionally samples the GPU through NVML (the GPU analogue of the Pi's CPU monitor)."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from colearn_federated_learning_b200.utils.monitors import main  # noqa: E402

if __name__ == "__main__":
    main()
