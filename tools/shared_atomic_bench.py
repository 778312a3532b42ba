"""Shared-memory atomic probe numbers of one GPU: per unit the kernel time of one launch (CUDA events) and the launches
a probe took, the host time spent on the expected words and the wall time of a default probe (medians over --reps
default probes), with the card's name and power limit read in the same run.

    python tools/shared_atomic_bench.py [--gpu 0] [--reps 10]
"""
import argparse
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from gpushare_device_plugin_b200 import _abi, device  # noqa: E402
from tools.copy_bench import card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpu", type=int, default=0)
    ap.add_argument("--reps", type=int, default=10)
    a = ap.parse_args()
    device.init()
    name, watts = card(a.gpu)
    uuid = device.device_info(a.gpu).uuid
    device.shared_atomic_probe(a.gpu)  # warm-up
    rs = [device.shared_atomic_probe(a.gpu) for _ in range(a.reps)]
    for r in rs:
        assert r.status == 0 and device.shared_atomic_conditions(r) == 0, device.shared_atomic_text(r, uuid)
    units = {}
    for u, uname in enumerate(_abi.SHARED_ATOMIC_UNIT_NAMES):
        units[uname] = {"kernel_us": round(statistics.median(r.run[u].kernel_ns / r.run[u].launches for r in rs) / 1e3, 1),
                        "launches": max(r.run[u].launches for r in rs),
                        "worst_cas_loop_us": round(max(r.run[u].cas_max_ns for r in rs) / 1e3, 1)}
    out = {
        "card": name, "power_limit_w": watts, "sm_count": rs[-1].sm_count, "reps": a.reps, "units": units,
        "expected_ms": round(statistics.median(r.expected_ns / 1e6 for r in rs), 2),
        "wall_ms_default": round(statistics.median(r.wall_ns / 1e6 for r in rs), 2),
    }
    print(json.dumps(out))
    print(device.shared_atomic_text(rs[-1], uuid))
    device.shutdown()


if __name__ == "__main__":
    main()
