"""Time GaussianProcess.predict_and_grad on the bench.py dense problem (N = 65536, 1.0 * ExpSquared(1.0), 3-D, diag
0.1) at M test points drawn over the same cube: predict_and_grad without the variance, with return_var=True, and
predict(return_var=True), alternating the three in one run on one factor.  Each call is timed by CUDA events around
it (every library call ends in a stream synchronisation); the library's profile timers give its phases: the kernel
builds (build), the forward substitution (forward), the backward substitution (backward) and the kernel-gradient
contraction with its reduction (contract).  predict(return_var=True) builds, substitutes and downdates the M x M
conditioned covariance and factors it, as the reference's predict does.

    python tools/predict_grad_bench.py [--n 65536] [--m 1024 16384] [--reps 2] [--out FILE]

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
    ap.add_argument("--m", type=int, nargs="+", default=[1024, 16384])
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch

    from bench import make_dense_problem
    from tinygp_b200 import GaussianProcess, _cabi, kernels

    if not torch.cuda.is_available():
        raise SystemExit("predict_grad_bench needs a GPU")
    X, y, diag, scale = make_dense_problem(args.n)
    side = float(X.max())
    gp = GaussianProcess(1.0 * kernels.ExpSquared(scale), X, diag=diag)
    ctx = _cabi.get_context()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    legs = {
        "grad": lambda Xt: gp.predict_and_grad(y, Xt),
        "grad_var": lambda Xt: gp.predict_and_grad(y, Xt, return_var=True),
        "predict_var": lambda Xt: gp.predict(y, Xt, return_var=True),
    }

    def timed(leg, Xt):
        ctx.set_option("profile", 1)
        ctx.profile(reset=True)
        torch.cuda.synchronize()
        ev[0].record()
        out = legs[leg](Xt)
        ev[1].record()
        torch.cuda.synchronize()
        p = ctx.profile(reset=True)
        ctx.set_option("profile", 0)
        phases = {"build": p["build_ms"] / 1e3, "forward": p["solve_ms"] / 1e3, "backward": p["bsolve_ms"] / 1e3,
                  "contract": p["contract_ms"] / 1e3}
        return out, ev[0].elapsed_time(ev[1]) / 1e3, phases

    gp.predict(y, X[:1])                      # the factorisation, outside every timed call
    res = {"workload": f"dense ExpSquared 3-D N={args.n}: predict_and_grad (without / with variance) and "
                       "predict(return_var=True) at M test points, alternating", "runs": {}}
    for m in args.m:
        Xt = np.random.default_rng(m).uniform(0.0, side, (m, 3))
        for leg in legs:                       # warm-up: module loads, buffer cache
            timed(leg, Xt)
        runs = {leg: [] for leg in legs}
        for _ in range(args.reps):             # alternate the legs so that drift of the shared card affects all
            for leg in legs:
                out, t, ph = timed(leg, Xt)
                runs[leg].append({"s": t, **{k + "_s": v for k, v in ph.items()}})
        mu, var, g = legs["grad_var"](Xt)
        mu_p, var_p = legs["predict_var"](Xt)
        res["runs"][str(m)] = {
            **runs,
            "mu_equal_predict": bool(np.array_equal(mu, mu_p)),
            "var_max_abs_diff": float(np.max(np.abs(var - var_p))),
            "dmean_norm": float(np.linalg.norm(g.mean)), "dvar_norm": float(np.linalg.norm(g.var)),
        }
    res["gpu"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                                capture_output=True, text=True).stdout.strip()
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
