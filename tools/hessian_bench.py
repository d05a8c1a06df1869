"""Time GaussianProcess.log_probability_hessian against fisher_information and log_probability_and_grad with CUDA
events, on the bench.py dense point set (3-D, the same point density at every N), for the P = 3 and P = 8 models of
tools/fisher_bench.py:

    P = 3:  c * ExpSquared(s), scalar diag
    P = 8:  c1 * ExpSquared(s1) + c2 * Matern32(s2) + c3 * RQ(s3, alpha), L2 distances, scalar diag

    python tools/hessian_bench.py [--n 16384] [--reps 2] [--out FILE]

The three calls alternate, so that drift of a shared card affects each.  Prints one JSON line; needs a GPU."""

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
    ap.add_argument("--n", type=int, nargs="+", default=[16384])
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch

    from bench import make_dense_problem
    from tinygp_b200 import GaussianProcess, kernels

    if not torch.cuda.is_available():
        raise SystemExit("hessian_bench needs a GPU")
    models = {
        3: lambda: 1.0 * kernels.ExpSquared(1.0),
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
            _, _, H = gp.log_probability_hessian(y)          # warm-up: module loads, buffer cache
            assert len(H.params) == rows and np.all(np.isfinite(H.matrix)), (H.params, H.matrix)
            gp.fisher_information()
            gp.log_probability_and_grad(y)
            t_h, t_f, t_g = [], [], []
            for _ in range(args.reps):
                (_, _, H), t = timed(lambda: gp.log_probability_hessian(y))
                t_h.append(t)
                _, t = timed(gp.fisher_information)
                t_f.append(t)
                _, t = timed(lambda: gp.log_probability_and_grad(y))
                t_g.append(t)
            runs.append({"n": n, "P": rows, "hessian_s": min(t_h), "fisher_s": min(t_f), "grad_s": min(t_g),
                         "hessian_minus_fisher_s": min(t_h) - min(t_f),
                         "hessian_over_fisher_plus_grad": min(t_h) / (min(t_f) + min(t_g)),
                         "all_hessian_s": t_h, "all_fisher_s": t_f, "all_grad_s": t_g,
                         "hessian_diag": H.matrix.diagonal().tolist()})
            print(json.dumps(runs[-1]), file=sys.stderr, flush=True)
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    line = json.dumps({"workload": "dense 3-D log_probability_hessian vs fisher_information and log_probability_and_grad",
                       "gpu": gpu, "runs": runs})
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
