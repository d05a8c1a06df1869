"""Rate of each fp64 tensor-core (DMMA) mma shape on this GPU: a register-resident loop of one shape on all SMs
(b200gp_measure_dmma_shape), burst (short loop, best of 3) and sustained (a loop of about a second or more, where a
power-limited card has settled its clocks).  Prints one JSON line with the card, its power limit and max SM clock.

    python tools/dmma_shapes.py [--sustained-iters 1500000]
"""

import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from tinygp_b200 import _cabi  # noqa: E402

SHAPES = [(8, 8, 4), (16, 8, 4), (16, 8, 8), (16, 8, 16)]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True).stdout.splitlines()[0]
    name, power, clock = (f.strip() for f in q.split(","))
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--burst-iters", type=int, default=4096)
    ap.add_argument("--sustained-iters", type=int, default=1_500_000)
    args = ap.parse_args()
    ctx = _cabi.get_context()
    out = {"card": card(), "unit": "TFLOP/s", "shapes": {}}
    try:
        for m, n, k in SHAPES:
            ctx.set_option("peak_iters", args.burst_iters)
            burst = max(ctx.measure_dmma_shape(m, n, k) for _ in range(3))
            ctx.set_option("peak_iters", args.sustained_iters)
            sustained = ctx.measure_dmma_shape(m, n, k)
            out["shapes"][f"m{m}n{n}k{k}"] = {"burst": burst, "sustained": sustained}
    finally:
        ctx.reset_options()
    base = out["shapes"]["m8n8k4"]["sustained"]
    out["sustained_vs_m8n8k4"] = {s: v["sustained"] / base for s, v in out["shapes"].items()}
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
