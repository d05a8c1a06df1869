"""Full-size LAPACK known answers for the bench workloads (one-off, N = 65 536).

    python tests/golden/make_golden_full.py c2      # N=65536 ExpSquared, the bench default (about 30 min, 35 GB)
    python tests/golden/make_golden_full.py c3s     # N=65537 Matern52+RationalQuadratic (L2), the sharded workload

Independent of oracle/ and of tinygp_b200/: the covariance is written out from the kernel definitions
(src/tinygp/kernels/stationary.py:104-106,150-153,232-235 with the Euclidean metric of kernels/distance.py:48-59,
explicit coordinate differences), factorised by a textbook blocked Cholesky over LAPACK/BLAS block calls and the log-density assembled as in
src/tinygp/gp.py:312-315 / solvers/direct.py:61-70.  NOT reference-produced (the reference needs JAX).  The inputs
are the bench's (bench.py make_dense_problem / run_sharded: same seeds and formulas), regenerated here.
Results go to tests/golden/full_size.json.
"""
import json
import os
import sys
import time

import numpy as np
from scipy.linalg import lapack, solve_triangular

HERE = os.path.dirname(os.path.abspath(__file__))


def problem(which):
    if which == "c2":
        n, seed, side0, n0 = 65536, 49382, 20.0, 65536.0
    elif which == "c3s":
        n, seed, side0, n0 = 65537, 49383, 25.0, 131072.0
    else:
        raise SystemExit("c2 | c3s")
    rng = np.random.default_rng(seed)
    side = side0 * (n / n0) ** (1.0 / 3.0)
    X = np.ascontiguousarray(rng.uniform(0.0, side, (n, 3)))
    y = np.sin(X[:, 0]) + 0.1 * rng.normal(size=n)
    return n, seed, X, y, 0.1


def cov_rows(which, Xa, Xb):
    r2 = np.zeros((Xa.shape[0], Xb.shape[0]))
    for d in range(3):
        df = Xa[:, d, None] - Xb[None, :, d]
        r2 += df * df
    if which == "c2":                      # 1.0 * ExpSquared(scale=1.0)
        return np.exp(-0.5 * r2)
    r = np.sqrt(r2)                        # 1.5 * Matern52(2.0, L2) + 0.7 * RationalQuadratic(1.5, L2, alpha=1.5)
    a = np.sqrt(5.0) * (r / 2.0)
    m52 = (1.0 + a + a * a / 3.0) * np.exp(-a)
    rq = (1.0 + 0.5 * (r2 / 1.5 ** 2) / 1.5) ** (-1.5)
    return 1.5 * m52 + 0.7 * rq


def main():
    which = sys.argv[1]
    n, seed, X, y, diag = problem(which)
    if len(sys.argv) > 2:                  # dry run at a reduced size (not written to the JSON)
        n = int(sys.argv[2])
        X, y = X[:n], y[:n]
    t0 = time.time()
    K = np.empty((n, n))                   # row-major; only the lower triangle is filled and read
    step = 1024
    for s in range(0, n, step):
        e = min(n, s + step)
        K[s:e, :e] = cov_rows(which, X[s:e], X[:e])
    K[np.diag_indices(n)] += diag
    t1 = time.time()
    # Textbook blocked right-looking Cholesky on the lower triangle, every LAPACK/BLAS call on a block of at most
    # n x NB doubles: one dpotrf over all 2^32 elements trips 32-bit element counts in the f2py/LAPACK stack (it
    # fails at n = 65536 and works at 16384, where this blocked form reproduces it to 1e-13).
    NB = 8192
    alpha = y.copy()
    logdet_half = 0.0
    for j in range(0, n, NB):
        e = min(n, j + NB)
        Ljj, info = lapack.dpotrf(K[j:e, j:e], lower=1, clean=1)
        assert info == 0, info
        K[j:e, j:e] = Ljj
        logdet_half += float(np.sum(np.log(np.diagonal(Ljj))))
        alpha[j:e] = solve_triangular(Ljj, alpha[j:e], lower=True, check_finite=False)
        if e < n:
            # panel: L[e:, j:e] = K[e:, j:e] Ljj^-T, block row by block row to bound the temporaries
            for i in range(e, n, NB):
                ie = min(n, i + NB)
                K[i:ie, j:e] = solve_triangular(Ljj, K[i:ie, j:e].T, lower=True, check_finite=False).T
            alpha[e:] -= K[e:, j:e] @ alpha[j:e]
            for i in range(e, n, NB):     # trailing update of the lower triangle only
                ie = min(n, i + NB)
                K[i:ie, e:ie] -= K[i:ie, j:e] @ K[e:ie, j:e].T
        print("block column", j, "done %.0f s" % (time.time() - t1), flush=True)
    t2 = time.time()
    logp = -0.5 * float(alpha @ alpha) - (logdet_half + 0.5 * n * np.log(2.0 * np.pi))
    if len(sys.argv) > 2:
        print(which, n, logp)
        return
    out_path = os.path.join(HERE, "full_size.json")
    out = json.load(open(out_path)) if os.path.exists(out_path) else {}
    out[which] = {"n": n, "seed": seed, "diag": diag, "log_probability": logp, "half_logdet": logdet_half,
                  "quad": float(alpha @ alpha), "x_checksum": float(X.sum()), "y_checksum": float(y.sum()),
                  "build_s": round(t1 - t0, 1), "dpotrf_s": round(t2 - t1, 1),
                  "lapack": "blocked (NB=8192) dpotrf/dtrsm/dgemm, scipy %s, %d threads" % (__import__("scipy").__version__, os.cpu_count())}
    json.dump(out, open(out_path, "w"), indent=1, sort_keys=True)
    print(which, out[which])


if __name__ == "__main__":
    main()
