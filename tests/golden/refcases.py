"""Reference-generated golden cases: one definition, three executors.

`run_case(ns, case)` drives a `GaussianProcess` API through the quantities it exposes.  The *same* kernel
expression strings are evaluated against

  * the unmodified reference (`tinygp` from /root/reference over tests/golden/jaxshim) -> make_golden_reference.py
    writes reference_vectors.json,
  * the oracle (`oracle.tinygp_np`)                        -> tests/test_reference_golden.py on CPU,
  * the product (`tinygp_b200`, CUDA through the C-ABI)    -> tests/test_reference_golden.py -m gpu,

which is also a statement about the drop-in surface: the names `kernels.*`, `kernels.quasisep.*`, `transforms.*`,
`GaussianProcess(...).log_probability / condition / predict` and the solver methods mean the same thing in all three.
"""

import numpy as np


class Namespace:
    """what a case may use: GaussianProcess, kernels, quasisep, transforms + three accessors that differ by backend"""

    def __init__(self, name, GaussianProcess, kernels, quasisep, transforms, qs_factor, to_np=np.asarray, noise=None):
        self.name, self.GaussianProcess, self.noise = name, GaussianProcess, noise
        self.kernels, self.quasisep, self.transforms = kernels, quasisep, transforms
        self.qs_factor, self.to_np = qs_factor, to_np

    def kernel(self, expr):
        env = {"kernels": self.kernels, "quasisep": self.quasisep, "transforms": self.transforms, "np": np}
        return eval(expr, env)  # noqa: S307 -- expressions are the literals in CASES below


def _inputs(case):
    rng = np.random.default_rng(case["seed"])
    n, m = case["n"], case.get("m", 7)
    if case["kind"] == "quasisep":
        t = np.sort(rng.uniform(0.0, case["span"], n))
        if case.get("ties"):
            t[5] = t[4]
            t[n // 2 + 1] = t[n // 2]
        y = np.sin(t) + 0.1 * rng.normal(size=n)
        tt = rng.uniform(-0.05 * case["span"], 1.05 * case["span"], m)   # unsorted, extrapolating on both sides
        tt[0] = t[3]                                                    # coincides with a datum
        z = rng.normal(size=n)
        return {"X": t, "y": y, "X_test": tt, "z": z, "y_test": np.cos(tt)}
    d = case["d"]
    X = rng.uniform(0.0, case["span"], (n, d))
    if d == 1:
        X = np.sort(X[:, 0]) if case.get("sorted") else X[:, 0]
    y = np.sin(X if d == 1 else X[:, 0]) + 0.1 * rng.normal(size=n)
    Xt = rng.uniform(0.0, case["span"], (m, d))
    if d == 1:
        Xt = Xt[:, 0]
    z = rng.normal(size=n)
    return {"X": X, "y": y, "X_test": Xt, "z": z, "y_test": np.cos(Xt if d == 1 else Xt[:, 0])}


# fmt: off
L2 = "distance=kernels.L2Distance()"
CASES = [
    # ---- dense (DirectSolver): BASELINE configs at oracle-friendly sizes, every stationary leaf, sums/products
    dict(name="c1_expsq_1d_n256", kind="dense", kernel="kernels.ExpSquared(scale=1.5)", n=256, d=1, span=6.0, sorted=True, diag=0.1, seed=84930),
    dict(name="c2_expsq_3d_n512", kind="dense", kernel="1.0 * kernels.ExpSquared(scale=1.0)", n=512, d=3, span=20.0 * (512 / 65536.0) ** (1 / 3.0), diag=0.1, seed=49382, small=False),
    dict(name="c3_m52_rq_L2_3d", kind="dense", kernel=f"1.5 * kernels.Matern52(2.0, {L2}) + 0.7 * kernels.RationalQuadratic(scale=1.5, {L2}, alpha=1.5)", n=300, d=3, span=25.0 * (300 / 131072.0) ** (1 / 3.0), diag=0.1, seed=49383),
    dict(name="c3_m52_rq_L1default_3d", kind="dense", kernel="1.5 * kernels.Matern52(2.0) + 0.7 * kernels.RationalQuadratic(scale=1.5, alpha=1.5)", n=300, d=3, span=25.0 * (300 / 131072.0) ** (1 / 3.0), diag=0.1, seed=49383),
    dict(name="m52_L1_3d_indefinite", kind="dense", kernel="kernels.Matern52(1.0)", n=400, d=3, span=6.0, diag=1e-3, seed=11, small=False),
    dict(name="exp_1d", kind="dense", kernel="0.9 * kernels.Exp(scale=1.3)", n=90, d=1, span=8.0, diag=0.05, seed=1),
    dict(name="m32_1d", kind="dense", kernel="kernels.Matern32(scale=0.7)", n=90, d=1, span=8.0, diag=0.05, seed=2),
    dict(name="m32_L2_2d", kind="dense", kernel=f"1.1 * kernels.Matern32(1.3, {L2})", n=90, d=2, span=5.0, diag=0.05, seed=3),
    dict(name="m52_1d_mean", kind="dense", kernel="0.8 * kernels.Matern52(1.1)", n=90, d=1, span=8.0, diag=0.05, seed=4, mean=0.3),
    dict(name="cosine_x_expsq_1d", kind="dense", kernel="kernels.Cosine(scale=2.5) * kernels.ExpSquared(scale=3.0)", n=90, d=1, span=8.0, diag=0.05, seed=5),
    dict(name="expsinesq_1d", kind="dense", kernel="1.3 * kernels.ExpSineSquared(scale=2.0, gamma=0.7)", n=90, d=1, span=8.0, diag=0.2, seed=6),
    dict(name="rq_L1_1d", kind="dense", kernel="kernels.RationalQuadratic(scale=1.5, alpha=0.8)", n=90, d=1, span=8.0, diag=0.05, seed=7),
    dict(name="combo_1d", kind="dense", kernel="1.2 * kernels.ExpSquared(0.7) + kernels.RationalQuadratic(1.5, alpha=1.5) * 0.5 + 0.05", n=90, d=1, span=8.0, diag=0.05, seed=8),
    dict(name="prod_sum_3d", kind="dense", kernel=f"(kernels.Matern32(1.3, {L2}) + 0.3) * kernels.ExpSquared(2.0) + 0.2 * kernels.Exp(1.7, {L2})", n=90, d=3, span=4.0, diag=0.05, seed=9),
    dict(name="default_jitter_1d", kind="dense", kernel="kernels.Matern32(scale=1.0)", n=60, d=1, span=12.0, diag=None, seed=10),
    dict(name="linear_scalar_1d", kind="dense", kernel="transforms.Linear(1 / 4.5, kernels.Matern32())", n=70, d=1, span=20.0, diag=0.05, seed=12),
    dict(name="linear_matrix_3d", kind="dense", kernel="transforms.Linear(np.array([[0.9, 0.1, 0.0], [0.0, 1.2, -0.3], [0.2, 0.0, 0.7]]), kernels.ExpSquared())", n=70, d=3, span=4.0, diag=0.05, seed=13),
    dict(name="cholesky_3d", kind="dense", kernel=f"transforms.Cholesky.from_parameters(np.array([1.1, 0.8, 1.4]), np.array([0.2, -0.1, 0.3]), kernels.Matern52({L2}))", n=70, d=3, span=4.0, diag=0.05, seed=14),
    dict(name="subspace_additive_3d", kind="dense", kernel="transforms.Subspace(0, kernels.ExpSquared(1.2)) + 0.5 * transforms.Subspace(np.array([1, 2]), kernels.Matern32(0.9))", n=70, d=3, span=4.0, diag=0.05, seed=15),
    # ---- BASELINE config 5: corners of the (scale, amplitude) hyper-parameter grid, same X ~ U(0, 8)^3 density
    dict(name="c5_grid_scale_lo_amp_lo", kind="dense", kernel="0.1 * kernels.ExpSquared(scale=10 ** -0.5)", n=128, d=3, span=8.0 * (128 / 4096.0) ** (1 / 3.0), diag=0.1, seed=49385),
    dict(name="c5_grid_scale_lo_amp_hi", kind="dense", kernel="10.0 * kernels.ExpSquared(scale=10 ** -0.5)", n=128, d=3, span=8.0 * (128 / 4096.0) ** (1 / 3.0), diag=0.1, seed=49385),
    dict(name="c5_grid_scale_hi_amp_lo", kind="dense", kernel="0.1 * kernels.ExpSquared(scale=10 ** 0.5)", n=128, d=3, span=8.0 * (128 / 4096.0) ** (1 / 3.0), diag=0.1, seed=49385),
    dict(name="c5_grid_scale_hi_amp_hi", kind="dense", kernel="10.0 * kernels.ExpSquared(scale=10 ** 0.5)", n=128, d=3, span=8.0 * (128 / 4096.0) ** (1 / 3.0), diag=0.1, seed=49385),
    # ---- quasiseparable (QuasisepSolver): BASELINE config 4 kernel, every state-space model, ties, both scan modes
    dict(name="c4_sho_m32_n200", kind="quasisep", kernel="quasisep.SHO(omega=1.5, quality=3.0, sigma=1.8) + quasisep.Matern32(scale=1.5, sigma=0.9)", n=200, span=20.0, diag=0.1, seed=49384),
    dict(name="c4_sho_m32_n200_parallel", kind="quasisep", kernel="quasisep.SHO(omega=1.5, quality=3.0, sigma=1.8) + quasisep.Matern32(scale=1.5, sigma=0.9)", n=200, span=20.0, diag=0.1, seed=49384, parallel=True),
    dict(name="sho_critical", kind="quasisep", kernel="quasisep.SHO(omega=1.2, quality=0.5, sigma=1.1)", n=120, span=30.0, diag=0.05, seed=21),
    dict(name="sho_overdamped", kind="quasisep", kernel="quasisep.SHO(omega=1.2, quality=0.2, sigma=1.1)", n=120, span=30.0, diag=0.05, seed=22),
    dict(name="qs_exp", kind="quasisep", kernel="quasisep.Exp(scale=1.7, sigma=0.8)", n=120, span=30.0, diag=0.05, seed=23),
    dict(name="qs_m32_ties", kind="quasisep", kernel="quasisep.Matern32(scale=1.5, sigma=1.8)", n=120, span=30.0, diag=0.05, seed=24, ties=True),
    dict(name="qs_m52", kind="quasisep", kernel="quasisep.Matern52(scale=2.5, sigma=1.3)", n=120, span=30.0, diag=0.05, seed=25),
    dict(name="qs_celerite", kind="quasisep", kernel="quasisep.Celerite(1.1, 0.1, 0.3, 1.5)", n=120, span=30.0, diag=0.05, seed=26),
    dict(name="qs_cosine_plus_exp", kind="quasisep", kernel="quasisep.Cosine(scale=3.0, sigma=0.7) + quasisep.Exp(scale=2.0, sigma=0.5)", n=120, span=30.0, diag=0.05, seed=27),
    dict(name="qs_scaled_sum3", kind="quasisep", kernel="2.0 * quasisep.Matern32(1.2) + quasisep.SHO(0.8, 4.0, 0.6) + 0.5 * quasisep.Exp(5.0)", n=120, span=30.0, diag=0.05, seed=28),
    dict(name="qs_product_sho_m32", kind="quasisep", kernel="quasisep.SHO(omega=1.5, quality=3.0, sigma=1.8) * quasisep.Matern32(scale=1.5, sigma=0.9)", n=120, span=30.0, diag=0.05, seed=29),
    dict(name="qs_scaled_product_plus_m52", kind="quasisep", kernel="0.7 * (quasisep.Exp(scale=2.0, sigma=1.1) * quasisep.Celerite(1.1, 0.1, 0.3, 1.5)) + quasisep.Matern52(scale=2.5, sigma=1.3)", n=120, span=30.0, diag=0.05, seed=30),
    # CARMA (kernels/quasisep.py:690-900): one real root + a complex pair; a complex pair; two real roots; one real root; in a sum
    dict(name="qs_carma31", kind="quasisep", kernel="quasisep.CARMA(alpha=np.array([1.4, 2.3, 1.5]), beta=np.array([0.1, 0.5]))", n=120, span=30.0, diag=0.05, seed=31),
    dict(name="qs_carma21_complex", kind="quasisep", kernel="quasisep.CARMA(alpha=np.array([1.0, 1.2]), beta=np.array([1.0, 3.0]))", n=120, span=30.0, diag=0.05, seed=32),
    dict(name="qs_carma21_real", kind="quasisep", kernel="quasisep.CARMA(alpha=np.array([0.1, 1.1]), beta=np.array([1.0, 3.0]))", n=120, span=30.0, diag=0.05, seed=33),
    dict(name="qs_carma10", kind="quasisep", kernel="quasisep.CARMA(alpha=np.array([1.0 / 100]), beta=np.array([0.3]))", n=120, span=30.0, diag=0.05, seed=34),
    dict(name="qs_carma_plus_m32", kind="quasisep", kernel="quasisep.CARMA.init(alpha=np.array([1.4, 2.3, 1.5]), beta=np.array([0.1, 0.5])) + 0.5 * quasisep.Matern32(1.5)", n=120, span=30.0, diag=0.05, seed=35),
    # 7 and 8 states; a Sum inside a Product (multiplied out by the host lowering: the state vector is a permutation of the
    # reference's, so only permutation-invariant outputs are recorded: small=False)
    dict(name="qs_product_m52_cosine_plus_exp_7", kind="quasisep", kernel="quasisep.Matern52(scale=2.5, sigma=1.3) * quasisep.Cosine(scale=3.0, sigma=0.7) + quasisep.Exp(scale=2.0, sigma=0.5)", n=120, span=30.0, diag=0.05, seed=51),
    dict(name="qs_m52_m52_sho_8", kind="quasisep", kernel="quasisep.Matern52(scale=2.5, sigma=1.3) + quasisep.Matern52(scale=0.6, sigma=0.4) + quasisep.SHO(omega=1.5, quality=3.0, sigma=0.8)", n=120, span=30.0, diag=0.05, seed=52),
    dict(name="qs_product_of_sum_8", kind="quasisep", kernel="(quasisep.Matern52(1.5) + 0.4 * quasisep.Exp(0.7)) * quasisep.SHO(omega=1.5, quality=0.1)", n=120, span=30.0, diag=0.05, seed=53, small=False),
    # noise.Banded / noise.Dense (noise.py:98-240): the precomputed-covariance paths of both solvers
    dict(name="qs_m32_sho_noise_banded2", kind="quasisep", kernel="quasisep.Matern32(scale=1.5, sigma=1.8) + quasisep.SHO(omega=1.2, quality=2.0, sigma=0.7)", n=120, span=30.0, seed=41, noise="banded", band=2),
    dict(name="qs_exp_noise_banded5", kind="quasisep", kernel="quasisep.Exp(scale=1.7, sigma=0.8)", n=120, span=30.0, seed=42, noise="banded", band=5),
    dict(name="m52_3d_noise_dense", kind="dense", kernel="0.8 * kernels.Matern52(1.1)", n=90, d=3, span=4.0, seed=43, noise="dense"),
    dict(name="expsq_1d_noise_banded3", kind="dense", kernel="1.2 * kernels.ExpSquared(0.7)", n=90, d=1, span=8.0, seed=44, noise="banded", band=3),
    dict(name="qs_scaled_sum3_parallel", kind="quasisep", kernel="2.0 * quasisep.Matern32(1.2) + quasisep.SHO(0.8, 4.0, 0.6) + 0.5 * quasisep.Exp(5.0)", n=120, span=30.0, diag=0.05, seed=28, parallel=True),
]
# fmt: on


def _noise(ns, case, n):
    """noise.Banded / noise.Dense (noise.py:98-240) instead of a diagonal: seeded, diagonally dominant"""
    rng = np.random.default_rng(case["seed"] + 7)
    diag = rng.uniform(0.1, 0.2, n)
    if case["noise"] == "banded":
        return ns.noise.Banded(diag=diag, off_diags=0.02 * rng.normal(size=(n, case.get("band", 2))))
    R = rng.normal(size=(n, 3))
    return ns.noise.Dense(value=np.diag(diag) + 0.02 * (R @ R.T))


def run_case(ns, case):
    """-> dict of float / list outputs.  `small` cases (default for n <= 120) also record full vectors."""
    inp = _inputs(case)
    X, y, Xt, z = inp["X"], inp["y"], inp["X_test"], inp["z"]
    k = ns.kernel(case["kernel"])
    kw = {}
    if case.get("diag") is not None:
        kw["diag"] = case["diag"]
    if "mean" in case:
        kw["mean"] = case["mean"]
    if case.get("parallel"):
        kw["parallel"] = True
    if "noise" in case:
        kw["noise"] = _noise(ns, case, case["n"])
    to_np = ns.to_np
    out = {}
    gp = ns.GaussianProcess(k, X, **kw)
    out["log_probability"] = float(to_np(gp.log_probability(y)))
    if not np.isfinite(out["log_probability"]):
        return out                                              # non-PD: the reference says -inf and nothing else is defined
    full = case.get("small", True) and case["n"] <= 120
    out["normalization"] = float(to_np(gp.solver.normalization()))
    var = to_np(gp.variance)
    out["variance_sum"] = float(np.sum(var))
    alpha = to_np(gp.solver.solve_triangular(y - to_np(gp.loc)))
    alpha_t = to_np(gp.solver.solve_triangular(alpha, transpose=True))
    dot = to_np(gp.solver.dot_triangular(z))
    out["alpha_norm"], out["alpha_t_norm"], out["dot_norm"] = (float(np.linalg.norm(v)) for v in (alpha, alpha_t, dot))
    cond = gp.condition(y, Xt, diag=1e-3)
    out["cond_log_probability"] = float(to_np(cond[0]))
    cgp = cond[1]
    out["pred_mean"] = to_np(cgp.loc).tolist()
    out["pred_var"] = to_np(cgp.variance).tolist()
    out["pred_cov_row0"] = to_np(cgp.covariance)[0].tolist()
    out["cond_gp_log_probability"] = float(to_np(cgp.log_probability(inp["y_test"])))
    cond_in = gp.condition(y, diag=0.05)                     # X_test=None branch (gp.py:340-346; solver.py:124-129)
    out["pred_in_mean_norm"] = float(np.linalg.norm(to_np(cond_in[1].loc)))
    out["pred_in_var_sum"] = float(np.sum(to_np(cond_in[1].variance)))
    cov_in = to_np(cond_in[1].covariance)
    out["pred_in_cov_trace"] = float(np.trace(cov_in))
    out["pred_in_cov_row0"] = cov_in[0, :8].tolist()
    out["cond_in_gp_log_probability"] = float(to_np(cond_in[1].log_probability(y + 0.01 * z)))
    mu_p, var_p = gp.predict(y, return_var=True)             # gp.py:225-271 at the inputs, default predictive jitter
    out["predict_in_mean_norm"] = float(np.linalg.norm(to_np(mu_p)))
    out["predict_in_var"] = to_np(var_p)[:: max(1, case["n"] // 16)].tolist()
    if case["kind"] == "dense":
        idx = np.arange(0, case["n"], max(1, case["n"] // 9))[:9]
        X1 = X[idx]
        out["K_cross"] = to_np(k(X1, Xt)).tolist()           # Kernel.__call__ two-argument form (base.py:89-103)
        out["K_diag"] = to_np(k(X1)).tolist()                # one-argument form -> diagonal (base.py:85-87)
    else:
        c, w = ns.qs_factor(gp)
        out["factor_c_sum_log"] = float(np.sum(np.log(c)))
        out["factor_w_norm"] = float(np.linalg.norm(w))
        out["matmul_norm"] = float(np.linalg.norm(to_np(k.matmul(X, y=z))))
        if full:
            out["factor_c"], out["factor_w"] = np.asarray(c).tolist(), np.asarray(w).tolist()
    if full:
        out["variance"] = var.tolist()
        out["alpha"], out["alpha_t"], out["dot"] = alpha.tolist(), alpha_t.tolist(), dot.tolist()
    return out
