"""``GaussianProcess`` re-declared without JAX (reference: src/tinygp/gp.py:30-393).

Same constructor and method signatures, so ``solver=`` drops in; all linear algebra goes through
the six ``Solver`` methods exactly where the reference calls them (gp.py:120,124,201,310,315,320,334).
"""

from __future__ import annotations

__all__ = ["GaussianProcess", "ConditionResult", "LogProbabilityGrad", "LogProbabilityGradX", "FisherInformation",
           "LogProbabilityHessian", "PredictionGrad"]

import copy
from typing import Any, NamedTuple

import numpy as np

from tinygp_b200 import kernels, means, transforms
from tinygp_b200.kernels.quasisep import Quasisep
from tinygp_b200.noise import Diagonal, Noise
from tinygp_b200.solvers import DirectSolver, QuasisepSolver
from tinygp_b200.solvers.quasisep.core import SymmQSM


class GaussianProcess:
    def __init__(self, kernel, X, *, diag=None, noise: Noise | None = None, mean=None, solver: Any | None = None,
                 mean_value=None, covariance_value: Any | None = None, **solver_kwargs: Any):
        self.kernel = kernel
        if isinstance(X, (dict, tuple)) or np.asarray(X).dtype == object or np.ndim(X) not in (1, 2):
            raise ValueError("coordinates must be an array of shape (N,) or (N, D); pytree coordinates (gp.py:40-44) "
                             "are unsupported by the B200 solver backend")
        self.X = X
        self._zero_mean = mean is None and mean_value is None      # default Mean(0.0): y - loc == y (skips an N-vector pass)
        if isinstance(mean, means.MeanBase):  # gp.py:81-86
            self.mean_function = mean
        elif mean is None:
            self.mean_function = means.Mean(0.0)
        else:
            self.mean_function = means.Mean(mean)
        if mean_value is None:
            mean_value = self.mean_function.vmap(self.X)  # gp.py:87-88
        mean_value = np.asarray(mean_value, dtype=np.float64)
        if mean_value.ndim != 1:
            raise ValueError(f"Invalid mean shape: expected ndim = 1, got ndim={mean_value.ndim}")
        self.num_data = mean_value.shape[0]
        self.dtype = mean_value.dtype
        self.mean = mean_value
        self._scalar_diag = noise is None and np.ndim(diag) == 0     # its gradient is then the sum over the diagonal
        if noise is None:  # gp.py:96-99
            diag = _default_diag(self.mean) if diag is None else diag
            noise = Diagonal(diag=_as_full_diag(diag, self.mean.shape))
        self.noise = noise
        if solver is None:  # gp.py:101-105
            solver = QuasisepSolver if (isinstance(covariance_value, SymmQSM) or isinstance(kernel, Quasisep)) else DirectSolver
        self.solver = solver(kernel, self.X, self.noise, covariance=covariance_value, **solver_kwargs)

    @property
    def loc(self):
        return self.mean

    @property
    def variance(self):
        return self.solver.variance()

    @property
    def covariance(self):
        return self.solver.covariance()

    def log_probability(self, y):  # gp.py:126-138
        hook = getattr(self.solver, "whitened_sumsq", None)
        if hook is not None:     # same value as below with |alpha|^2 reduced on the device (no N-vector round trip)
            with np.errstate(all="ignore"):
                yv = np.asarray(y, dtype=np.float64)
                loglike = -0.5 * hook(yv if self._zero_mean else yv - self.loc) - self.solver.normalization()
            return loglike if np.isfinite(loglike) else -np.inf
        return self._compute_log_prob(self._get_alpha(y))

    def log_probability_and_grad(self, y, *, wrt_X: bool = False):
        """``log_probability(y)`` and its exact gradient with respect to the kernel parameters, the noise diagonal and
        the mean, from one device call: the factor, L^-1 in place, and the contraction of (alpha alpha^T - K^-1) with
        dK/dtheta evaluated tile by tile (W = K^-1 is never stored).  Needs the dense DirectSolver, a diagonal noise
        model, and a kernel made of stationary leaves, Constant, sums, products and 0- / 1-D transforms.Linear /
        Cholesky and Subspace, with at most 16 differentiable scalars; anything else raises NotImplementedError.  A
        non positive-definite covariance gives (-inf, NaN gradients).  The solver's own factor is not touched.

        Returns ``(logp, LogProbabilityGrad)``; with ``wrt_X=True``, ``(logp, LogProbabilityGradX)``, which also holds
        d logp / d X with the shape of X, from the same device call (at most 8 input dimensions).  Only the kernel's
        dependence on X is differentiated: a mean *function* of X is not, and ``grad.mean`` (d logp / d mean) is there to
        chain through it.  At coincident points the kernel's gradient is taken as 0."""
        hook = getattr(self.solver, "log_probability_grad", None)
        if hook is None:
            raise NotImplementedError(f"log_probability_and_grad: no gradients for {type(self.solver).__name__} (only "
                                      "the dense DirectSolver)")
        yv = np.asarray(y, dtype=np.float64)
        resid = yv if self._zero_mean else yv - self.loc
        if wrt_X:
            logp, grads, ddiag, alpha, dX = hook(resid, wrt_X=True)
        else:
            logp, grads, ddiag, alpha = hook(resid)
        if not np.isfinite(logp):
            logp = -np.inf
        fields = dict(kernel=_grad_tree(self.kernel, grads, {}),
                      diag=float(np.sum(ddiag)) if self._scalar_diag else ddiag, mean=alpha)
        if wrt_X:
            return logp, LogProbabilityGradX(**fields, X=dX.reshape(np.shape(self.X)))
        return logp, LogProbabilityGrad(**fields)

    def fisher_information(self) -> "FisherInformation":
        """The expected Fisher information of ``log_probability`` with respect to the kernel's differentiable fields and
        a scalar ``diag``: F_ab = 1/2 tr(K^-1 dK/da K^-1 dK/db), which does not depend on y.  One device call: the factor,
        L^-1 in place, then for each parameter b the matrix K^-1 dK/db K^-1 by four triangular products and its
        contraction with every dK/da.  Its rows and columns are ``params``, the order in which ``log_probability_and_grad``
        visits the kernel (``FisherInformation.flatten`` reads a gradient in that order), then ``("diag", None)`` when
        ``diag`` was given as a scalar.  A per-point noise diagonal is not a parameter of F, and neither is the mean.

        Scope and refusals are those of ``log_probability_and_grad``: the dense DirectSolver, a diagonal noise model, at
        most 16 differentiable scalars; anything else raises NotImplementedError.  A node that occurs twice gets the sum
        over its occurrences.  A non positive-definite covariance gives an all-NaN matrix.  The solver's own factor is not
        touched.  Costs about 4 P n^3 flops and one n x n fp64 buffer beyond the gradient's memory (P the device's
        parameter count).  A Fisher-scoring step is ``np.linalg.solve(F.matrix, F.flatten(grad))``."""
        hook = getattr(self.solver, "fisher_information", None)
        if hook is None:
            raise NotImplementedError(f"fisher_information: not available for {type(self.solver).__name__} (only the "
                                      "dense DirectSolver)")
        Fs, rows = hook(self._scalar_diag)
        params, column, J = self._slot_jacobian(rows, Fs.shape[0])
        if not np.all(np.isfinite(Fs)):
            return FisherInformation(np.full((len(params), len(params)), np.nan), params)
        A = J.T @ Fs @ J
        return FisherInformation(0.5 * (A + A.T), params)

    def log_probability_hessian(self, y):
        """``log_probability(y)``, its gradient and its Hessian with respect to the kernel's differentiable fields and a
        scalar ``diag``, from one device call: the observed curvature at y, what ``jax.hessian`` of the log-likelihood
        gives (``fisher_information()`` is its expectation over y, with the sign flipped).  With W = K^-1 and
        alpha = W (y - mean):
            H_ab = 1/2 <alpha alpha^T - W, d2K/dadb> - (dK/da alpha)^T W (dK/db alpha) + 1/2 tr(W dK/da W dK/db)
        Returns ``(logp, LogProbabilityGrad, LogProbabilityHessian)``; the first two are those of
        ``log_probability_and_grad(y)``.  The Hessian's rows are ``params`` as in ``fisher_information``; fields that
        reach the kernel through a row scale of a transform (1-D ``Linear.scale`` / ``Cholesky.factor``) carry the
        curvature of that map too.  A Newton step is ``theta - np.linalg.solve(H.matrix, H.flatten(grad))`` in the
        order of ``params``, and ``np.linalg.inv(-H.matrix)`` at the maximum is the Laplace covariance.

        Scope and refusals are those of ``log_probability_and_grad``.  A non positive-definite covariance gives
        (-inf, NaN gradients, an all-NaN matrix).  The solver's own factor is not touched.  Costs the Fisher
        information's time and memory plus the second derivatives of the kernel, n^2 / 2 evaluations per pair of
        device parameters."""
        hook = getattr(self.solver, "log_probability_hessian", None)
        if hook is None:
            raise NotImplementedError(f"log_probability_hessian: not available for {type(self.solver).__name__} (only "
                                      "the dense DirectSolver)")
        yv = np.asarray(y, dtype=np.float64)
        resid = yv if self._zero_mean else yv - self.loc
        logp, grads, ddiag, alpha, Hs, rows, curvature = hook(resid, self._scalar_diag)
        if not np.isfinite(logp):
            logp = -np.inf
        grad = LogProbabilityGrad(kernel=_grad_tree(self.kernel, grads, {}),
                                  diag=float(np.sum(ddiag)) if self._scalar_diag else ddiag, mean=alpha)
        params, column, J = self._slot_jacobian(rows, Hs.shape[0])
        if not np.all(np.isfinite(Hs)):
            return logp, grad, LogProbabilityHessian(np.full((len(params), len(params)), np.nan), params)
        A = J.T @ Hs @ J
        for ka, kb, v in curvature:
            A[column[ka], column[kb]] += v
        return logp, grad, LogProbabilityHessian(0.5 * (A + A.T), params)

    def _slot_jacobian(self, rows, nslot):
        """(params, column, J) of fisher_information / log_probability_hessian: the parameter labels, the column of each
        (id(node), field, index), and J = d slot / d parameter from the solver's slot rows (plus the scalar diag last)"""
        entries = list(_param_walk(self.kernel))
        params = [label for label, _ in entries]
        column = {key: p for p, (_, key) in enumerate(entries)}
        if self._scalar_diag:
            params.append(("diag", None))
        J = np.zeros((nslot, len(params)))      # d slot / d parameter
        for s, ents in enumerate(rows):
            for node, field, idx, coef in ents:
                J[s, column[(id(node), field, idx)]] += coef
        if self._scalar_diag:
            J[-1, -1] = 1.0
        return params, column, J

    def condition(self, y, X_test=None, *, diag=None, noise: Noise | None = None, include_mean: bool = True,
                  kernel=None) -> "ConditionResult":
        """gp.py:140-223"""
        self._check_X_test(X_test)
        alpha, log_prob, mean_value = self._condition(y, X_test, include_mean, kernel)
        if kernel is None:
            kernel = self.kernel
        if noise is None:
            diag = _default_diag(mean_value) if diag is None else diag
            noise = Diagonal(diag=np.broadcast_to(np.asarray(diag, dtype=np.float64), mean_value.shape).copy())
        cond_kernel = kernels.Conditioned(self.X, self.solver, kernel)
        cond_mean = means.Conditioned(self.X, alpha, kernel, include_mean=include_mean, mean_function=self.mean_function)
        covariance_value = self.solver.condition(kernel, X_test, noise)  # gp.py:201
        if X_test is None:
            X_test = self.X
        gp = GaussianProcess(  # gp.py:208-221: the conditional GP factors the M x M covariance again
            cond_kernel,
            X_test,
            noise=noise,
            mean=cond_mean,
            mean_value=mean_value,
            covariance_value=covariance_value,
            # a SymmQSM (solver.py:124-129) is factored in O(N) by QuasisepSolver(covariance=...), gp.py:101-103
            solver=None if isinstance(covariance_value, SymmQSM) else DirectSolver,
        )
        return ConditionResult(log_prob, gp)

    def predict(self, y, X_test=None, *, kernel=None, include_mean: bool = True, return_var: bool = False,
                return_cov: bool = False):
        """gp.py:225-271.  The reference's ``predict`` is jitted with ``return_var`` / ``return_cov`` static
        (gp.py:225-229), so XLA never computes the conditioned covariance when only the mean is asked for; the same
        holds here explicitly -- the mean needs ``alpha`` and one kernel product, not ``solver.condition`` (which for a
        quasiseparable N = 10^7 series would be an N x N matrix)."""
        if not (return_var or return_cov):
            self._check_X_test(X_test)
            return self._condition(y, X_test, include_mean, kernel)[2]
        if return_var and X_test is None and kernel is None and getattr(self.solver, "conditioned_variance", None) is not None:
            # QuasisepSolver at the inputs: the reference's QSM branch (solver.py:124-129) keeps this O(N); so does the
            # backward scan behind conditioned_variance -- same values as cond.variance below
            mean_value = self._condition(y, None, include_mean, None)[2]
            noise = Diagonal(diag=np.full(mean_value.shape, _default_diag(mean_value)))
            return mean_value, self.solver.conditioned_variance(noise)
        _, cond = self.condition(y, X_test, kernel=kernel, include_mean=include_mean)
        if return_var:
            return cond.loc, cond.variance
        if return_cov:
            return cond.loc, cond.covariance
        return cond.loc

    def predict_and_grad(self, y, X_test, *, kernel=None, include_mean: bool = True, return_var: bool = False):
        """``predict(y, X_test, ...)`` and its gradient with respect to the test inputs: ``(mu, PredictionGrad)``, or
        ``(mu, var, PredictionGrad)`` with ``return_var=True``.  ``kernel`` and ``include_mean`` mean what they mean in
        ``predict``.  ``mu`` is bit for bit ``predict(y, X_test, kernel=kernel, include_mean=include_mean)`` (the same
        computation); ``var`` is ``predict(..., return_var=True)[1]`` up to the rounding of its sum of squares:
        k(x*, x*) + sqrt(eps) - |L^-1 k(X, x*)|^2, the default predictive noise included.

        With alpha = K^-1 (y - mean) and v_m = K^-1 k(X, x*_m), the device computes
            d mu_m / d x*_m  = sum_j grad_1 k(x*_m, x_j) alpha_j,
            d var_m / d x*_m = -2 sum_j grad_1 k(x*_m, x_j) v_m,j
        in one call on the solver's own factor (built first if still pending; no second one).  mu_m and var_m depend on
        X_test[m] only, so ``PredictionGrad.mean`` / ``.var`` (the shape of X_test) are the only non-zero blocks of the
        Jacobians.  A mean *function* of X_test is not differentiated (as ``LogProbabilityGradX.X``): with a callable
        mean, ``mean`` is the ``include_mean=False`` gradient.  At a test point that coincides with a training point the
        pair's kernel gradient is taken as 0 (exact for the smooth kernels).

        Scope and refusals are those of ``log_probability_and_grad(wrt_X=True)``, for the predictive kernel: the dense
        DirectSolver built from a kernel program with a diagonal noise model, stationary leaves, Constant, sums,
        products, 0- / 1-D transforms.Linear / Cholesky and Subspace, at most 16 differentiable scalars and 8 input
        dimensions; anything else raises NotImplementedError.  A failed factorisation does not raise: the arrays are NaN.
        The variance costs about 2 n^2 M flops of triangular solves on top of the mean's n M kernel-gradient
        evaluations, and at most one 4096 x n fp64 buffer."""
        hook = getattr(self.solver, "predict_grad", None)
        if hook is None:
            raise NotImplementedError(f"predict_and_grad: no gradients for {type(self.solver).__name__} (only the dense "
                                      "DirectSolver)")
        if X_test is None:
            raise ValueError("predict_and_grad: X_test is required")
        self._check_X_test(X_test)
        alpha, _, mu = self._condition(y, X_test, include_mean, kernel)
        diag = np.full(np.shape(mu), _default_diag(mu)) if return_var else None
        dmean, var, dvar = hook(self.kernel if kernel is None else kernel, X_test, alpha, diag)
        shape = np.shape(X_test)
        grad = PredictionGrad(mean=dmean.reshape(shape), var=None if dvar is None else dvar.reshape(shape))
        return (mu, var, grad) if return_var else (mu, grad)

    def sample(self, key, shape=None):
        """gp.py:273-311.  ``key`` seeds numpy's Generator (JAX's threefry stream is not reproducible
        without JAX -- sample-value parity is statistical only, as in tests/test_gp.py:24-38)."""
        rng = key if isinstance(key, np.random.Generator) else np.random.default_rng(key)
        shape = (self.num_data,) if shape is None else (self.num_data,) + tuple(shape)
        normal_samples = rng.standard_normal(shape)
        return self.mean + np.moveaxis(self.solver.dot_triangular(normal_samples), 0, -1)

    def _check_X_test(self, X_test):  # gp.py:180-191
        if X_test is not None:
            a, b = np.asarray(self.X), np.asarray(X_test)
            if a.ndim != b.ndim or a.shape[1:] != b.shape[1:]:
                raise ValueError(
                    "`X_test` must have the same tree structure as the input `X`, "
                    "and all but the leading dimension must have matching sizes"
                )

    # -- internals (gp.py:313-361) -------------------------------------------------------------
    def _compute_log_prob(self, alpha):
        with np.errstate(all="ignore"):
            loglike = -0.5 * np.sum(np.square(alpha)) - self.solver.normalization()
        return loglike if np.isfinite(loglike) else -np.inf

    def _get_alpha(self, y):
        return self.solver.solve_triangular(np.asarray(y, dtype=np.float64) - self.loc)

    def _condition(self, y, X_test, include_mean, kernel=None):
        y = np.asarray(y, dtype=np.float64)
        alpha = self._get_alpha(y)
        log_prob = self._compute_log_prob(alpha)
        alpha = self.solver.solve_triangular(alpha, transpose=True)  # gp.py:334
        if X_test is None:
            if kernel is None:
                delta = self.noise @ alpha  # gp.py:342-346
                mean_value = y - delta
                if not include_mean:
                    mean_value = mean_value - self.loc
            else:
                mean_value = kernel.matmul(self.X, y=alpha)
                if include_mean:
                    mean_value = mean_value + self.loc
        else:
            if kernel is None:
                kernel = self.kernel
            mean_value = kernel.matmul(X_test, self.X, alpha)  # gp.py:357
            if include_mean:
                mean_value = mean_value + self.mean_function.vmap(X_test)
        return alpha, log_prob, mean_value


class ConditionResult(NamedTuple):
    """gp.py:364-385"""
    log_probability: Any
    gp: GaussianProcess


class LogProbabilityGrad(NamedTuple):
    """Gradient of ``GaussianProcess.log_probability``: ``kernel`` is a structural copy of the kernel whose
    differentiable fields (Constant.value, Stationary.scale, ExpSineSquared.gamma, RationalQuadratic.alpha, 0- / 1-D
    Linear.scale and Cholesky.factor) hold d logp / d field, and whose other fields are None -- what ``jax.grad`` returns
    for an equinox module; a node that occurs twice holds the sum.  ``diag``: d logp / d diag (a float for a scalar
    ``diag``, else one value per point); ``mean``: d logp / d mean = K^-1 (y - mean)."""
    kernel: Any
    diag: Any
    mean: np.ndarray


class LogProbabilityGradX(NamedTuple):
    """``LogProbabilityGrad`` and ``X``: d logp / d X through the kernel, with the shape of the coordinates ((N,) or
    (N, D)), from ``log_probability_and_grad(y, wrt_X=True)``.  A mean function of X is not differentiated: chain
    ``mean`` (= d logp / d mean) through it."""
    kernel: Any
    diag: Any
    mean: np.ndarray
    X: np.ndarray


class PredictionGrad(NamedTuple):
    """Gradient of ``GaussianProcess.predict`` with respect to the test inputs, from ``predict_and_grad``: ``mean``
    holds d mu_m / d X_test[m] and ``var`` d var_m / d X_test[m] (None unless ``return_var=True``), both with the shape
    of X_test ((M,) or (M, D)).  mu_m and var_m depend on X_test[m] only, so these are the only non-zero blocks of the
    Jacobians.  A mean function of X_test is not differentiated."""
    mean: np.ndarray
    var: Any


class FisherInformation(NamedTuple):
    """``GaussianProcess.fisher_information()``: ``matrix`` (P x P, float64, symmetric bit for bit) over ``params``, one
    label per row: ``(path, None)`` for a scalar field, e.g. ``("kernel1.value", None)``, ``(path, i)`` for entry i of a
    1-D ``Linear.scale`` / ``Cholesky.factor``, e.g. ``("kernel2.kernel.scale", 1)``, and ``("diag", None)`` last for a
    scalar ``diag``."""
    matrix: np.ndarray
    params: list

    def flatten(self, grad) -> np.ndarray:
        """a ``LogProbabilityGrad`` (or ``LogProbabilityGradX``) of the same model as a vector in ``params`` order"""
        return _flatten(self.params, grad, "Fisher information")


class LogProbabilityHessian(NamedTuple):
    """``GaussianProcess.log_probability_hessian(y)``: ``matrix`` (P x P, float64, symmetric bit for bit), the Hessian of
    ``log_probability`` at y over ``params``, labelled and ordered as ``FisherInformation.params``."""
    matrix: np.ndarray
    params: list

    def flatten(self, grad) -> np.ndarray:
        """a ``LogProbabilityGrad`` (or ``LogProbabilityGradX``) of the same model as a vector in ``params`` order"""
        return _flatten(self.params, grad, "Hessian")


def _flatten(params, grad, what):
    entries = list(_param_walk(grad.kernel, values=True))
    labels = [label for label, _ in entries]
    has_diag = bool(params) and params[-1] == ("diag", None)
    if labels != list(params[:len(params) - has_diag]):
        raise ValueError(f"flatten: the gradient's kernel does not have this {what}'s parameters")
    out = [value for _, value in entries]
    if has_diag:
        if np.ndim(grad.diag) != 0:
            raise ValueError(f"flatten: the {what} has a scalar diag, the gradient a per-point one")
        out.append(float(grad.diag))
    return np.asarray(out, dtype=np.float64)


def _param_walk(node, values=False, path="", memo=None):
    """(label, key) of every differentiable scalar in the order _grad_tree visits the kernel: depth-first over
    vars(node), a shared node once, one entry per index of a 1-D field; key = (id(node), field, index or None), or with
    ``values`` the field's value there"""
    memo = set() if memo is None else memo
    if id(node) in memo:
        return
    memo.add(id(node))
    fields = _grad_fields(node)
    for name, value in vars(node).items():
        label = path + name
        if isinstance(value, kernels.Kernel):
            yield from _param_walk(value, values, label + ".", memo)
        elif name in fields:
            if np.ndim(value) == 0:
                yield (label, None), (float(value) if values else (id(node), name, None))
            else:
                flat = np.asarray(value, dtype=np.float64).reshape(-1)
                for i in range(flat.shape[0]):
                    yield (label, i), (float(flat[i]) if values else (id(node), name, i))


def _grad_fields(node) -> tuple[str, ...]:
    if isinstance(node, kernels.Constant):
        return ("value",)
    if isinstance(node, kernels.Stationary):
        return ("scale",) + ((node.p1_field,) if node.p1_field else ())
    if isinstance(node, transforms.Linear):
        return ("scale",)
    if isinstance(node, transforms.Cholesky):
        return ("factor",)
    return ()


def _grad_tree(node, grads, memo):
    if id(node) in memo:
        return memo[id(node)]
    out = copy.copy(node)
    memo[id(node)] = out
    fields = _grad_fields(node)
    got = grads.get(id(node), (None, {}))[1]
    for name, value in vars(node).items():
        if isinstance(value, kernels.Kernel):
            setattr(out, name, _grad_tree(value, grads, memo))
        elif name in fields:
            shape = np.shape(value)
            g = got.get(name, np.zeros(shape) if shape else 0.0)
            setattr(out, name, float(g) if not shape else np.asarray(g, dtype=np.float64))
        else:
            setattr(out, name, None)
    return out


def _as_full_diag(diag, shape):
    """jnp.broadcast_to(diag, shape) of gp.py:98; an array that already has the full shape is passed through as it is (no
    copy: a caller's page-locked buffer stays page-locked all the way to the device copy)"""
    d = np.asarray(diag, dtype=np.float64)
    if d.shape == tuple(shape) and d.flags.c_contiguous:
        return d
    return np.broadcast_to(d, shape).copy()


def _default_diag(reference):  # gp.py:388-393
    return np.sqrt(np.finfo(np.asarray(reference).dtype).eps)
