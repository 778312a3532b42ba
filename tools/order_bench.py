"""Memory-ordering probe numbers of one GPU: per unit the kernel time of one launch (CUDA events), its overlap count
(observations that saw a partner mid-stream) and MP_RELAXED's weak outcomes, the wall time of a default probe (medians
over --reps default probes), with the card's name and power limit read in the same run.

    python tools/order_bench.py [--gpu 0] [--reps 10] [--observations 1024]
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
    ap.add_argument("--observations", type=int, default=0)
    a = ap.parse_args()
    device.init()
    name, watts = card(a.gpu)
    uuid = device.device_info(a.gpu).uuid
    device.order_probe(a.gpu, observations=a.observations)  # warm-up
    rs = [device.order_probe(a.gpu, observations=a.observations) for _ in range(a.reps)]
    for r in rs:
        assert r.status == 0 and device.order_conditions(r) == 0, device.order_text(r, uuid)
    units = {}
    for u, uname in enumerate(_abi.ORDER_UNIT_NAMES):
        ran = [r.unit[u].kernel_ns / r.unit[u].launches for r in rs if r.unit[u].launches]  # every launch refused: none
        units[uname] = {"kernel_us": round(statistics.median(ran) / 1e3, 1) if ran else None,
                        "overlap": statistics.median(r.unit[u].overlap for r in rs),
                        "weak": statistics.median(r.unit[u].weak for r in rs),
                        "refused": sum(r.unit[u].refused for r in rs)}
    out = {"card": name, "power_limit_w": watts, "sm_count": rs[-1].sm_count, "reps": a.reps,
           "observations": rs[-1].observations, "units": units,
           "wall_ms_default": round(statistics.median(r.wall_ns / 1e6 for r in rs), 2)}
    print(json.dumps(out))
    print(device.order_text(rs[-1], uuid))
    device.shutdown()


if __name__ == "__main__":
    main()
