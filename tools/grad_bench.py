"""Time GaussianProcess.log_probability_and_grad against log_probability on the bench.py dense problem (N = 65536,
1.0 * ExpSquared(1.0), 3-D, diag 0.1) with CUDA events, and split the gradient call into its phases with the library's
profile timers: factorisation (build + panels + trailing update), triangular inverse, contraction.

    python tools/grad_bench.py [--n 65536] [--reps 2] [--out FILE]

By flop count a gradient costs about 3x a log_probability (N^3 / 3 each for the factor, the inverse and the
contraction); what the card reaches is measured here.  Prints one JSON line; needs a GPU."""

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
        raise SystemExit("grad_bench needs a GPU")
    X, y, diag, scale = make_dense_problem(args.n)
    kern = 1.0 * kernels.ExpSquared(scale)
    ctx = _cabi.get_context()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]

    def timed(fn):
        torch.cuda.synchronize()
        ev[0].record()
        out = fn()                       # every library call returns after a stream synchronisation
        ev[1].record()
        torch.cuda.synchronize()
        return out, ev[0].elapsed_time(ev[1]) / 1e3

    lp = lambda: GaussianProcess(kern, X, diag=diag).log_probability(y)
    gr = lambda: GaussianProcess(kern, X, diag=diag).log_probability_and_grad(y)
    lp(), gr()                           # warm-up: module loads, buffer cache
    t_lp, t_gr, phases = [], [], []
    for _ in range(args.reps):           # alternate the two so that drift of the shared card affects both
        v_lp, t = timed(lp)
        t_lp.append(t)
        ctx.set_option("profile", 1)
        ctx.profile(reset=True)
        (v_gr, g), t = timed(gr)
        p = ctx.profile(reset=True)
        ctx.set_option("profile", 0)
        t_gr.append(t)
        phases.append({"factor_s": (p["syrk_ms"] + p["panel_ms"] + p["build_ms"]) / 1e3, "solve_s": p["solve_ms"] / 1e3,
                       "inverse_s": p["trtri_ms"] / 1e3, "contraction_s": p["contract_ms"] / 1e3})
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    n = args.n
    res = {
        "workload": f"dense ExpSquared 3-D N={n}: log_probability_and_grad vs log_probability",
        "gpu": gpu, "log_probability_s": min(t_lp), "log_probability_and_grad_s": min(t_gr),
        "ratio": min(t_gr) / min(t_lp), "phases_of_fastest_grad": phases[int(np.argmin(t_gr))],
        "all_log_probability_s": t_lp, "all_grad_s": t_gr,
        "flop_inverse_plus_contraction": 2.0 * n**3 / 3.0,
        "logp": v_lp, "logp_from_grad_call": v_gr,
        "grad": {"amp": g.kernel.kernel1.value, "scale": g.kernel.kernel2.scale, "diag_sum": float(np.sum(g.diag))},
    }
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
