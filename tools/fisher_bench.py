"""Time GaussianProcess.fisher_information against log_probability_and_grad with CUDA events, on the bench.py dense
point set (3-D, the same point density at every N), for P = 3 and P = 8 rows of F:

    P = 3:  c * ExpSquared(s), scalar diag                                  (2 kernel slots + diag)
    P = 8:  c1 * ExpSquared(s1) + c2 * Matern32(s2) + c3 * RQ(s3, alpha), L2 distances, scalar diag   (7 + diag)

    python tools/fisher_bench.py [--n 16384 32768] [--reps 2] [--out FILE]

The achieved rate counts the flops of the tile schedules the call runs: the factor (N^3 / 3), the triangular inverse
(TRMM and its panel products) and 4 P products by L^-1 (128^3 T^2 (T + 1) each, T = N / 128); the contraction's
derivative evaluations are not counted.  The denominator is the sustained fp64 DMMA rate that b200gp_measure_fp64_peak
measures on the same card.  Prints one JSON line; needs a GPU."""

import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

TILE = 128


def schedule_flops(n, rows):
    """flops of the factor, the inverse and the 4 * rows products by L^-1 for N = n"""
    T = -(-n // TILE)
    blk = 2.0 * TILE**3
    inverse = sum((T - 1 - j) + sum(ti - j for ti in range(j + 1, T)) for j in range(T - 1)) * blk
    products = 4 * rows * TILE**3 * T * T * (T + 1)
    return (T * TILE) ** 3 / 3.0 + inverse + products


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, nargs="+", default=[16384, 32768])
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch

    from bench import make_dense_problem
    from tinygp_b200 import GaussianProcess, _cabi, kernels

    if not torch.cuda.is_available():
        raise SystemExit("fisher_bench needs a GPU")
    ctx = _cabi.get_context()
    ctx.set_option("peak_iters", 1_500_000)
    peak = ctx.measure_fp64_peak()[0]
    ctx.reset_options()
    models = {
        3: lambda: 1.0 * kernels.ExpSquared(1.0),
        # L2 distances: Matern32 and RationalQuadratic on the default L1 distance are not positive definite in 3-D
        8: lambda: (1.0 * kernels.ExpSquared(1.0) + 0.5 * kernels.Matern32(2.0, distance=kernels.L2Distance())
                    + 0.3 * kernels.RationalQuadratic(1.5, distance=kernels.L2Distance(), alpha=1.2)),
    }
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]

    def timed(fn):
        torch.cuda.synchronize()
        ev[0].record()
        out = fn()                       # every library call returns after a stream synchronisation
        ev[1].record()
        torch.cuda.synchronize()
        return out, ev[0].elapsed_time(ev[1]) / 1e3

    runs = []
    for n in args.n:
        X, y, _, _ = make_dense_problem(n)
        for rows, make in models.items():
            gp = GaussianProcess(make(), X, diag=0.1)
            F = gp.fisher_information()          # warm-up: module loads, buffer cache
            assert len(F.params) == rows and np.all(np.isfinite(F.matrix)), (F.params, F.matrix)
            gp.log_probability_and_grad(y)
            t_f, t_g = [], []
            for _ in range(args.reps):       # alternate the two so that drift of the shared card affects both
                F, t = timed(gp.fisher_information)
                t_f.append(t)
                _, t = timed(lambda: gp.log_probability_and_grad(y))
                t_g.append(t)
            flops = schedule_flops(n, rows)
            runs.append({"n": n, "P": rows, "fisher_s": min(t_f), "grad_s": min(t_g), "ratio": min(t_f) / min(t_g),
                         "schedule_tflop": flops / 1e12, "tflops": flops / min(t_f) / 1e12,
                         "share_of_measured_dmma_peak": flops / min(t_f) / 1e12 / peak,
                         "all_fisher_s": t_f, "all_grad_s": t_g, "fisher_diag": F.matrix.diagonal().tolist()})
            print(json.dumps(runs[-1]), file=sys.stderr, flush=True)
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    line = json.dumps({"workload": "dense 3-D fisher_information vs log_probability_and_grad", "gpu": gpu,
                       "measured_dmma_peak_tflops": peak, "runs": runs})
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
