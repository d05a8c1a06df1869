"""Developer harness for a gpurun call: micro-benchmarks, parity spot checks and timing sweeps.
Writes gpurun_out/dev_<tag>.json.  Not part of the product or the tests."""

import json
import os
import sys
import time
from ctypes import byref, c_double

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import tinygp_np as o  # noqa: E402
from tinygp_b200 import _cabi, kernels  # noqa: E402

out = {}
ctx = _cabi.get_context()
tag = sys.argv[1] if len(sys.argv) > 1 else "run"
sizes = [int(s) for s in (sys.argv[2].split(",") if len(sys.argv) > 2 else "4096,16384,32768,65536".split(","))]
nbs = [int(s) for s in (sys.argv[3].split(",") if len(sys.argv) > 3 else "512".split(","))]
slices_list = [int(s) for s in (sys.argv[4].split(",") if len(sys.argv) > 4 else "0".split(","))]
clusters = [int(s) for s in (sys.argv[5].split(",") if len(sys.argv) > 5 else "22".split(","))]
lookaheads = [int(s) for s in (sys.argv[6].split(",") if len(sys.argv) > 6 else "1".split(","))]

if os.environ.get("LAYOUT"):
    ctx.set_option("ozaki_layout", int(os.environ["LAYOUT"]))
if os.environ.get("PAIRING"):
    ctx.set_option("ozaki_pairing", int(os.environ["PAIRING"]))
if os.environ.get("PREFETCH"):
    ctx.set_option("ozaki_prefetch", int(os.environ["PREFETCH"]))
out["fp64_peak"] = [ctx.measure_fp64_peak() for _ in range(1)]
print("fp64 peak (dmma, dfma) TF/s:", out["fp64_peak"], flush=True)


def logp_dev(n, nb, profile, slices=0):
    rng = np.random.default_rng(49382)
    X = np.ascontiguousarray(rng.uniform(0, 20.0 * (n / 65536.0) ** (1 / 3), (n, 3)))
    y = np.sin(X[:, 0]) + 0.1 * rng.normal(size=n)
    diag = np.full(n, 0.1)
    k = 1.0 * kernels.ExpSquared(1.0)
    prog = k.program()
    ctx.set_option("nb", nb)
    ctx.set_option("ozaki_slices", slices)
    ctx.set_option("ozaki_min_n", 0)
    ctx.set_option("profile", int(profile))
    ctx.profile(reset=True)
    lp = c_double()
    t0 = time.perf_counter()
    ctx.check(ctx.lib.b200gp_dense_log_probability(ctx.handle, _cabi.ptr(prog), prog.shape[0], _cabi.ptr(X), n, 3,
                                                   _cabi.ptr(diag), _cabi.ptr(y), byref(lp)))
    dt = time.perf_counter() - t0
    prof = ctx.profile(reset=True)
    ctx.set_option("profile", 0)
    return lp.value, dt, prof, (X, y)


res = []
for n in sizes:
  oracle_cache = {}
  for sl, cl, la in [(a, b, c) for a in slices_list for b in (clusters if a else [22]) for c in (lookaheads if a else [1])]:
    ctx.set_option("ozaki_cluster", cl)
    ctx.set_option("ozaki_lookahead", la)
    for nb in nbs:
        lp, dt, _, _ = logp_dev(n, nb, False, sl)       # warm-up (allocations)
        lp, dt, _, data = logp_dev(n, nb, False, sl)
        lp2, dt2, prof, _ = logp_dev(n, nb, True, sl)
        tf = n**3 / 3 / dt / 1e12
        row = {"n": n, "nb": nb, "slices": sl, "cluster": cl, "lookahead": la, "logp": lp, "sec": dt, "tflops_n3_3": tf, "profile": prof,
               "syrk_tflops": prof["syrk_flop"] / max(prof["syrk_ms"], 1e-9) / 1e9}
        if n <= 16384:
            X, y = data
            if n not in oracle_cache:
                t0 = time.perf_counter()
                lpo = o.GaussianProcess(o.Constant(1.0) * o.ExpSquared(1.0), X, diag=0.1).log_probability(y)
                oracle_cache[n] = (lpo, time.perf_counter() - t0)
            lpo, row["oracle_sec"] = oracle_cache[n]
            row["oracle_logp"] = lpo
            row["rel_err"] = abs(lp - lpo) / abs(lpo)
        print(json.dumps(row), flush=True)
        res.append(row)
out["dense"] = res
os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
json.dump(out, open(os.path.join(ROOT, "gpurun_out", f"dev_{tag}.json"), "w"), indent=1)
