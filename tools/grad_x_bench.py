"""Time GaussianProcess.log_probability_and_grad(y) against log_probability_and_grad(y, wrt_X=True) on the bench.py
dense problem (N = 65536, 1.0 * ExpSquared(1.0), 3-D, diag 0.1), alternating the two in one run, with CUDA events; the
library's profile timer gives the contraction phase (mirror, W tiles with their derivative epilogue, reductions) of
each, which is where the coordinate gradient is computed.

    python tools/grad_x_bench.py [--n 65536] [--reps 2] [--out FILE]

Prints one JSON line; needs a GPU."""

import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=65536)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch

    from bench import make_dense_problem
    from tinygp_b200 import GaussianProcess, _cabi, kernels

    if not torch.cuda.is_available():
        raise SystemExit("grad_x_bench needs a GPU")
    X, y, diag, scale = make_dense_problem(args.n)
    kern = 1.0 * kernels.ExpSquared(scale)
    ctx = _cabi.get_context()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]

    def timed(wrt_X):
        ctx.set_option("profile", 1)
        ctx.profile(reset=True)
        torch.cuda.synchronize()
        ev[0].record()
        out = GaussianProcess(kern, X, diag=diag).log_probability_and_grad(y, wrt_X=wrt_X)
        ev[1].record()
        torch.cuda.synchronize()             # every library call returns after a stream synchronisation
        p = ctx.profile(reset=True)
        ctx.set_option("profile", 0)
        return out, ev[0].elapsed_time(ev[1]) / 1e3, p["contract_ms"] / 1e3

    timed(False), timed(True)                # warm-up: module loads, buffer cache
    runs = {False: [], True: []}
    for _ in range(args.reps):               # alternate the two so that drift of the shared card affects both
        for wrt_X in (False, True):
            (lp, g), t, c = timed(wrt_X)
            runs[wrt_X].append((t, c, lp, g))
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    (_, _, lp0, g0), (_, _, lp1, g1) = runs[False][-1], runs[True][-1]
    res = {
        "workload": f"dense ExpSquared 3-D N={args.n}: log_probability_and_grad with and without wrt_X, alternating",
        "gpu": gpu,
        "grad_s": [r[0] for r in runs[False]], "grad_x_s": [r[0] for r in runs[True]],
        "grad_contract_s": [r[1] for r in runs[False]], "grad_x_contract_s": [r[1] for r in runs[True]],
        "logp_equal": lp0 == lp1, "diag_grad_equal": bool(np.array_equal(g0.diag, g1.diag)),
        "scale_grad_equal": g0.kernel.kernel2.scale == g1.kernel.kernel2.scale,
        "dX_norm": float(np.linalg.norm(g1.X)), "dX_sum_norm": float(np.linalg.norm(g1.X.sum(axis=0))),
        "dX_partials_bytes": (args.n // 128) * (args.n // 128 + 1) // 2 * 2 * 128 * X.shape[1] * 8,
    }
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
