"""B200 DirectSolver: same six-method contract as src/tinygp/solvers/direct.py:17-95, every method
bound to a C-ABI entry point of libb200gp.so.  The factor lives in HBM for the object's lifetime."""

from __future__ import annotations

__all__ = ["DirectSolver"]

from ctypes import byref, c_double, c_int, c_void_p
from typing import Any

import numpy as np

from tinygp_b200 import _cabi
from tinygp_b200.kernels.base import OP_ADD, OP_MUL, Kernel, Lowering
from tinygp_b200.noise import Diagonal
from tinygp_b200.solvers.solver import ConditionedCovariance, Solver


MAX_GRAD_SLOTS = 16     # differentiable scalars per kernel program (KGRAD_MAX_SLOTS, tinygp_b200/csrc/kgrad.cuh)
MAX_GRAD_DIM = 8        # input dimensions of gradients with respect to X (KGRAD_MAX_DIM, tinygp_b200/csrc/kgrad.cuh)


def _through_row_scale(value, s, kind):
    """``value`` per unit of a slot, carried to the field that moves it: unchanged where the slot is the field (kind
    None); through a row scale lambda, value * d lambda / d s_r = value / s_r (Linear), -value / f_r (Cholesky), and 0
    where s_r = 0"""
    if kind is None:
        return value
    if s == 0.0:
        return 0.0
    return value / s if kind == "linear" else -value / s


class DirectSolver(Solver):
    """Dense build fused into a blocked Cholesky on the fp64 tensor pipe (direct.py:30-53)."""

    def __init__(self, kernel: Kernel, X, noise, *, covariance: Any | None = None):
        self._ctx = _cabi.get_context()
        self._h = c_void_p()
        self.X = X
        self.kernel = kernel
        self.noise = noise
        self._pending = None
        self._info = 0
        info = c_int(0)
        lib = self._ctx.lib
        if covariance is None and not isinstance(noise, Diagonal):
            # noise.Dense / noise.Banded (direct.py:47-48: covariance = kernel(X, X) + noise): the kernel matrix is built on
            # the device, the noise matrix joins it on its way to the device factorisation of a precomputed covariance
            covariance = noise + kernel(X, X)
        if covariance is None and hasattr(kernel, "_has_closed_form") and not kernel._has_closed_form():
            # a user-defined quasiseparable model (kernels/quasisep.py:60-100 written in Python) has no kernel program: its
            # covariance comes from the device QSM algebra over host-evaluated generators (Quasisep._host_dense)
            covariance = noise + kernel(X, X)
        if covariance is None:
            prog, x = kernel.lower_for(X)   # x = X, plus host-computed columns of any transforms.Transform
            diag = _cabi.f64(noise.diagonal())
            if diag.shape != (x.shape[0],):
                raise ValueError("noise diagonal must have shape (N,)")
            self._n = x.shape[0]
            self._diag = diag
            self._x = x                      # the lowered (possibly transform-augmented) coordinates held on the device
            self.variance_value = kernel(X) + diag                              # direct.py:49
            self._cov = None
            # The factorisation (direct.py:53) is issued by the first method that needs it.  When that method is
            # `whitened_sumsq` -- GaussianProcess(...).log_probability(y), the benchmark's end-to-end path -- it runs as ONE
            # call that also substitutes the residual, panel by panel under the int8 update (b200gp_dense_create_with_resid);
            # any other first use factors alone (b200gp_dense_create).  Results are the same either way.
            self._pending = (prog, diag)
            return
        else:
            cov = _cabi.f64(covariance)
            if cov.ndim != 2 or cov.shape[0] != cov.shape[1]:
                raise ValueError("covariance must be a square matrix")
            self._n = cov.shape[0]
            self._x = None
            self._cov = cov
            # direct.py:49: variance = kernel(X) + noise.diagonal() with kernel = kernels.Conditioned, whose diagonal is
            # diag(Kss - A^T A).  DirectSolver.condition put the noise into Kss (direct.py:88-92) so that is diag(cov);
            # QuasisepSolver.condition's dense branch leaves it out (solvers/quasisep/solver.py:131-139), and the
            # reference's conditioned variance then still carries it (golden: reference_vectors.json pred_var).
            self.variance_value = np.diag(cov).copy()
            if not getattr(covariance, "includes_noise", True):    # solvers.solver.ConditionedCovariance tag
                self.variance_value = self.variance_value + _cabi.f64(noise.diagonal())
            self._ctx.check(lib.b200gp_dense_create_from_cov(self._ctx.handle, _cabi.ptr(cov), cov.shape[0],
                                                             byref(self._h), byref(info)))
        self._info = info.value

    @property
    def info(self):
        """0, or the 1-based index of the first non-positive pivot (the factor is NaN from there on, like
        jnp.linalg.cholesky's)"""
        self._ensure()
        return self._info

    def _ensure(self, resid=None):
        """factor now if that has not happened yet; with `resid` also return sum((L^-1 resid)^2) from the same pass"""
        if self._pending is None:
            return None
        prog, diag = self._pending
        x, info, lib = self._x, c_int(0), self._ctx.lib
        out = None
        if resid is None:
            self._ctx.check(lib.b200gp_dense_create(self._ctx.handle, _cabi.ptr(prog), prog.shape[0], _cabi.ptr(x),
                                                    x.shape[0], x.shape[1], _cabi.ptr(diag), byref(self._h), byref(info)))
        else:
            ss = c_double()
            self._ctx.check(lib.b200gp_dense_create_with_resid(self._ctx.handle, _cabi.ptr(prog), prog.shape[0], _cabi.ptr(x),
                                                               x.shape[0], x.shape[1], _cabi.ptr(diag), _cabi.ptr(resid),
                                                               byref(self._h), byref(info), byref(ss)))
            out = ss.value
        self._pending = None
        self._info = info.value
        return out

    def whitened_sumsq(self, y):
        """``sum(solve_triangular(y) ** 2)`` (the data term of gp.py:313-316).  Optional hook read by
        GaussianProcess.log_probability: on a solver that has not factored yet, factorisation and forward substitution are one
        device pass; afterwards it is the ordinary triangular solve."""
        y = _cabi.f64(y)
        if y.shape != (self._n,):
            raise ValueError("dimension mismatch")
        if self._pending is not None:
            return self._ensure(resid=y)
        return float(np.sum(np.square(self.solve_triangular(y))))

    def log_probability_grad(self, resid, wrt_X=False):
        """log_probability and its gradient for the residual ``resid = y - mean`` in one device call
        (b200gp_dense_log_probability_grad), with a factor of its own: the solver's factor, built or pending, is left
        as it is.  Returns (logp, grads, d logp / d diag, alpha) where ``grads`` maps id(node) to (node, {field:
        d logp / d field}) for every kernel node with a differentiable field reached by the program.  ``wrt_X``: one
        call of b200gp_dense_log_probability_grad_x instead, and a fifth item, d logp / d X of shape (N, D) (D = 1 for
        scalar coordinates), for at most MAX_GRAD_DIM input dimensions."""
        prog, x, slots = self._grad_slots("log_probability_and_grad")
        resid = _cabi.f64(resid)
        if resid.shape != (self._n,):
            raise ValueError("dimension mismatch")
        if wrt_X:
            if x.shape[1] > MAX_GRAD_DIM:
                raise NotImplementedError(f"log_probability_and_grad(wrt_X=True): the coordinates have {x.shape[1]} "
                                          f"dimensions; gradients with respect to X support at most {MAX_GRAD_DIM}")
            xu = np.asarray(self.X, dtype=np.float64)
            if x.shape != (self._n, 1 if xu.ndim == 1 else xu.shape[1]) or not np.array_equal(x.reshape(xu.shape), xu):
                # only transforms.Transform(callable) appends columns, and lower_for_grad refuses it
                raise AssertionError("log_probability_and_grad(wrt_X=True): the device coordinates differ from X")
        logp = c_double()
        dprog = np.zeros_like(prog)
        dmetric = np.zeros((Lowering.MAX_METRICS, Lowering.MAX_DIM))
        ddiag, alpha = np.empty(self._n), np.empty(self._n)
        args = (self._ctx.handle, _cabi.ptr(prog), prog.shape[0], _cabi.ptr(x), x.shape[0], x.shape[1],
                _cabi.ptr(self._diag), _cabi.ptr(resid), byref(logp), _cabi.ptr(dprog), _cabi.ptr(dmetric),
                _cabi.ptr(ddiag), _cabi.ptr(alpha))
        if wrt_X:
            dX = np.empty(x.shape)
            self._ctx.check(self._ctx.lib.b200gp_dense_log_probability_grad_x(*args, _cabi.ptr(dX)))
        else:
            self._ctx.check(self._ctx.lib.b200gp_dense_log_probability_grad(*args))
        grads: dict[int, tuple[Any, dict]] = {}

        def add(node, field, value, index=None):
            ent = grads.setdefault(id(node), (node, {}))[1]
            shape = np.shape(getattr(node, field))
            g = ent.setdefault(field, np.zeros(shape) if shape else 0.0)
            if index is None or not shape:
                ent[field] = g + value
            else:
                g[index] += value

        for (on, a, b), ents in slots:
            R = (dprog if on == 0 else dmetric)[a, b]
            for node, field, idx, s, kind in ents:
                add(node, field, _through_row_scale(R, s, kind), idx)
        if wrt_X:
            return logp.value, grads, ddiag, alpha, dX
        return logp.value, grads, ddiag, alpha

    def fisher_information(self, with_diag: bool):
        """The expected Fisher information over the device's slots (b200gp_dense_fisher), with a factor of its own: the
        solver's factor, built or pending, is left as it is.  ``with_diag``: one more slot, last, for a scalar noise
        diagonal (dK / d diag = I).  Returns (F, rows): F of shape (S + with_diag, S + with_diag), and for each program
        slot s the list rows[s] of (node, field, index, d slot / d field) that map it to the kernel's fields (index None
        for a scalar field) -- the slot-to-field map of log_probability_grad."""
        prog, x, slots = self._grad_slots("fisher_information")
        ns = c_int()
        origin = np.zeros(3 * MAX_GRAD_SLOTS, dtype=np.int32)
        F = np.empty((MAX_GRAD_SLOTS + 1) ** 2)
        self._ctx.check(self._ctx.lib.b200gp_dense_fisher(self._ctx.handle, _cabi.ptr(prog), prog.shape[0], _cabi.ptr(x),
                                                          x.shape[0], x.shape[1], _cabi.ptr(self._diag), int(bool(with_diag)),
                                                          byref(ns), _cabi.ptr(origin), _cabi.ptr(F)))
        if origin[:3 * ns.value].reshape(-1, 3).tolist() != [list(at) for at, _ in slots]:
            raise AssertionError("fisher_information: the device's slots differ from the host's slot map")
        k = ns.value + int(bool(with_diag))
        F = F[:k * k].reshape(k, k).copy()
        rows = [[(node, field, idx, _through_row_scale(1.0, s, kind)) for node, field, idx, s, kind in ents]
                for _, ents in slots]
        return F, rows

    def log_probability_hessian(self, resid, with_diag: bool):
        """log_probability_grad and the Hessian of logp over the device's slots from one device call
        (b200gp_dense_log_probability_hessian), with a factor of its own: the solver's factor, built or pending, is left
        as it is.  Returns (logp, grads, ddiag, alpha, H, rows, curvature): the first four as log_probability_grad
        returns them (bitwise the same values); H of shape (S + with_diag, S + with_diag), the noise diagonal last;
        rows as fisher_information returns them; and curvature, the terms that the slot map's own second derivatives
        add to the Hessian over the fields: (key_a, key_b, value) with key = (id(node), field, index), value = d logp /
        d slot times d^2 slot / d field_a d field_b.  A slot that is a row scale lambda = prod_k lambda_k of a chain of
        transforms has d^2 lambda / d p_k d p_l = (d lambda_k / d p_k) (d lambda_l / d p_l) for k != l, and d^2 lambda_k /
        d p_k^2 = 0 for Linear (lambda = s' / s), 2 / f^2 for Cholesky (lambda = f / f'; 0 where f = 0)."""
        prog, x, slots = self._grad_slots("log_probability_hessian")
        resid = _cabi.f64(resid)
        if resid.shape != (self._n,):
            raise ValueError("dimension mismatch")
        logp = c_double()
        dprog = np.zeros_like(prog)
        dmetric = np.zeros((Lowering.MAX_METRICS, Lowering.MAX_DIM))
        ddiag, alpha = np.empty(self._n), np.empty(self._n)
        ns = c_int()
        origin = np.zeros(3 * MAX_GRAD_SLOTS, dtype=np.int32)
        Hs = np.empty((MAX_GRAD_SLOTS + 1) ** 2)
        self._ctx.check(self._ctx.lib.b200gp_dense_log_probability_hessian(
            self._ctx.handle, _cabi.ptr(prog), prog.shape[0], _cabi.ptr(x), x.shape[0], x.shape[1], _cabi.ptr(self._diag),
            _cabi.ptr(resid), int(bool(with_diag)), byref(logp), _cabi.ptr(dprog), _cabi.ptr(dmetric), _cabi.ptr(ddiag),
            _cabi.ptr(alpha), byref(ns), _cabi.ptr(origin), _cabi.ptr(Hs)))
        if origin[:3 * ns.value].reshape(-1, 3).tolist() != [list(at) for at, _ in slots]:
            raise AssertionError("log_probability_hessian: the device's slots differ from the host's slot map")
        k = ns.value + int(bool(with_diag))
        Hs = Hs[:k * k].reshape(k, k).copy()
        grads: dict[int, tuple[Any, dict]] = {}

        def add(node, field, value, index=None):
            ent = grads.setdefault(id(node), (node, {}))[1]
            shape = np.shape(getattr(node, field))
            g = ent.setdefault(field, np.zeros(shape) if shape else 0.0)
            if index is None or not shape:
                ent[field] = g + value
            else:
                g[index] += value

        rows, curvature = [], []
        for (on, a, b), ents in slots:
            R = (dprog if on == 0 else dmetric)[a, b]
            for node, field, idx, s, kind in ents:
                add(node, field, _through_row_scale(R, s, kind), idx)
            rows.append([(node, field, idx, _through_row_scale(1.0, s, kind)) for node, field, idx, s, kind in ents])
            if on == 1:
                for ka, (na, fa, ia, sa, kinda) in enumerate(ents):
                    for kb, (nb, fb, ib, _, _) in enumerate(ents):
                        if ka != kb:
                            v = R * rows[-1][ka][3] * rows[-1][kb][3]
                        elif kinda == "cholesky" and sa != 0.0:
                            v = R * 2.0 / (sa * sa)
                        else:
                            continue
                        curvature.append(((id(na), fa, ia), (id(nb), fb, ib), v))
        return logp.value, grads, ddiag, alpha, Hs, rows, curvature

    def predict_grad(self, kernel: Kernel, X_test, alpha, diag_test=None):
        """d mu / d X_test of the predictive mean ``kernel.matmul(X_test, X, alpha)`` and, with ``diag_test`` (one
        predictive noise value per test point), the predictive variance and d var / d X_test, from one device call
        (b200gp_dense_predict_grad) on the solver's own factor, built first if it is still pending.  ``alpha`` =
        K^-1 (y - mean).  Returns (dmean, var, dvar): dmean and dvar of shape (M, D) (D = 1 for scalar coordinates),
        var of shape (M,); var and dvar are None without ``diag_test``.  The refusals are those of
        ``log_probability_and_grad(wrt_X=True)``, applied to the predictive kernel, plus the lowering check of
        ``condition``; messages name predict_and_grad."""
        who = "predict_and_grad"
        _, x, _ = self._grad_slots(who, kernel)
        if x.shape != self._x.shape or not np.array_equal(x, self._x):
            raise NotImplementedError(f"{who}: the predictive kernel lowers the training coordinates differently from the "
                                      "solver's kernel")
        if x.shape[1] > MAX_GRAD_DIM:
            raise NotImplementedError(f"{who}: the coordinates have {x.shape[1]} dimensions; gradients with respect to "
                                      f"X_test support at most {MAX_GRAD_DIM}")
        prog, xt = kernel.lower_for(X_test)
        if xt.shape[1] != x.shape[1]:
            raise ValueError("X_test must have the same number of input dimensions as the training inputs")
        alpha = _cabi.f64(alpha)
        if alpha.shape != (self._n,):
            raise ValueError("dimension mismatch")
        self._ensure()
        m = xt.shape[0]
        dmean = np.empty(xt.shape)
        var = dvar = None
        if diag_test is not None:
            diag_test = _cabi.f64(diag_test)
            if diag_test.shape != (m,):
                raise ValueError("noise diagonal must match the number of test points")
            var, dvar = np.empty(m), np.empty(xt.shape)
        ptr = lambda a: None if a is None else _cabi.ptr(a)
        self._ctx.check(self._ctx.lib.b200gp_dense_predict_grad(self._h, _cabi.ptr(prog), prog.shape[0], _cabi.ptr(xt), m,
                                                                _cabi.ptr(alpha), _cabi.ptr(dmean), ptr(diag_test),
                                                                ptr(var), ptr(dvar)))
        return dmean, var, dvar

    def _grad_slots(self, who: str, kernel: Kernel | None = None):
        """The refusals of log_probability_grad and fisher_information, messages prefixed by ``who``, and the slot map of
        ``lower_for_grad``: (prog, x, slots), one entry per device slot in kgrad_prepare's order (each leaf's p0 then
        p1 in program order, then the metric rows).  An entry is (where, fields): ``where`` is the slot's place in
        dprog / dmetric, (0, program row, 2 or 3) or (1, metric, row); ``fields`` lists the (node, field, index, s,
        kind) the slot moves, index None for a scalar field, kind None where the slot is the field itself, else the
        row-scale kind with s = field[index] (_through_row_scale).  ``kernel``: that kernel on the training inputs
        instead of the solver's."""
        if self._x is None:
            what = ("noise.Dense / noise.Banded" if not isinstance(self.noise, Diagonal)
                    else "a precomputed covariance (covariance=) or a kernel without a device program")
            raise NotImplementedError(f"{who}: not available for {what}; only kernel programs with a diagonal noise "
                                      "model are differentiated on the device")
        try:
            prog, x, leaves, owners = (self.kernel if kernel is None else kernel).lower_for_grad(self.X)
        except NotImplementedError as e:
            raise NotImplementedError(f"{who}: {e}") from e
        n_instr = 2 * len(leaves) - 1      # leaves and the binary ADD / MUL over them, after the metric rows
        ops = prog[-n_instr:, 0]
        leaf_rows = prog.shape[0] - n_instr + np.flatnonzero((ops != OP_ADD) & (ops != OP_MUL))
        slots = []
        for (node, f0, f1), row in zip(leaves, leaf_rows.tolist()):
            slots += [((0, row, 2 + c), [(node, f, None, None, None)]) for c, f in enumerate((f0, f1)) if f is not None]
        for m, chains in enumerate(owners):
            for r, chain in enumerate(chains):
                ents = []
                for node, field, idx, kind in chain:
                    v = np.asarray(getattr(node, field), dtype=np.float64)
                    idx = None if v.ndim == 0 else idx
                    ents.append((node, field, idx, float(v if idx is None else v[idx]), kind))
                slots.append(((1, m, r), ents))
        if len(slots) > MAX_GRAD_SLOTS:
            raise NotImplementedError(f"{who}: the kernel has {len(slots)} differentiable scalars (leaf scales, constants, "
                                      f"gamma / alpha, transform rows); at most {MAX_GRAD_SLOTS} are supported")
        return prog, x, slots

    def __del__(self):
        h = getattr(self, "_h", None)
        if h:
            try:
                self._ctx.lib.b200gp_dense_free(h)
            except Exception:
                pass
            self._h = c_void_p()

    # -- the Solver contract --------------------------------------------------------------
    def variance(self):
        return self.variance_value

    def covariance(self):  # direct.py:58-59, regenerated lazily by the build kernel
        if self._cov is None:
            self._ensure()
            out = np.empty((self._n, self._n))
            self._ctx.check(self._ctx.lib.b200gp_dense_covariance(self._h, _cabi.ptr(out)))
            self._cov = out
        return self._cov

    @property
    def scale_tril(self):
        self._ensure()
        out = np.empty((self._n, self._n))
        self._ctx.check(self._ctx.lib.b200gp_dense_get_factor(self._h, _cabi.ptr(out)))
        return out

    def normalization(self):  # direct.py:61-64
        self._ensure()
        ld = c_double()
        self._ctx.check(self._ctx.lib.b200gp_dense_logdet_half(self._h, byref(ld)))
        if self._info != 0:
            return np.nan
        return ld.value + 0.5 * self._n * np.log(2 * np.pi)

    def solve_triangular(self, y, *, transpose: bool = False):  # direct.py:66-70
        y = np.asarray(y, dtype=np.float64)
        if y.shape[0] != self._n:
            raise ValueError("dimension mismatch")
        self._ensure()
        buf = np.array(y.reshape(self._n, -1), dtype=np.float64, order="C", copy=True)
        self._ctx.check(self._ctx.lib.b200gp_dense_solve_triangular(self._h, _cabi.ptr(buf), buf.shape[1],
                                                                    int(bool(transpose))))
        return buf.reshape(y.shape)

    def dot_triangular(self, y):  # direct.py:72-73
        y = np.asarray(y, dtype=np.float64)
        if y.shape[0] != self._n:
            raise ValueError("dimension mismatch")
        self._ensure()
        buf = np.array(y.reshape(self._n, -1), dtype=np.float64, order="C", copy=True)
        self._ctx.check(self._ctx.lib.b200gp_dense_dot_triangular(self._h, _cabi.ptr(buf), buf.shape[1]))
        return buf.reshape(y.shape)

    def condition(self, kernel: Kernel, X_test, noise) -> Any:  # direct.py:75-95
        diag = _cabi.f64(noise.diagonal())
        if self._x is None:
            # a factor of a precomputed covariance (noise.Dense / noise.Banded, or a conditioned process) has no kernel
            # program on the device: direct.py:75-95 call by call -- Ks and Kss from the build kernel, A from the blocked
            # substitution, Kss - A^T A from the fp64 GEMM behind b200gp_gram_downdate
            Xs = self.X if X_test is None else X_test
            A = self.solve_triangular(kernel(self.X, Xs))
            out = np.ascontiguousarray(noise + kernel(Xs, Xs))
            At = np.ascontiguousarray(A.T)
            self._ctx.check(self._ctx.lib.b200gp_gram_downdate(self._ctx.handle, _cabi.ptr(At), At.shape[0], At.shape[1],
                                                               _cabi.ptr(out)))
            return ConditionedCovariance.tag(out, True)
        # b200gp_dense_condition evaluates the predictive kernel on the TRAINING coordinates kept on the device, i.e. in
        # the training kernel's lowered layout (raw columns + the host-computed columns of any transforms.Transform).
        # A predictive kernel that lowers the training inputs differently (other width, other transform outputs) would
        # read those columns wrongly -- or past the test-point buffer -- so it is refused instead of silently mis-evaluated.
        self._ensure()
        prog, x_train = kernel.lower_for(self.X)
        if x_train.shape != self._x.shape or not np.array_equal(x_train, self._x):
            raise NotImplementedError(
                f"the predictive kernel lowers the training coordinates to shape {x_train.shape} but the solver holds "
                f"{self._x.shape} (general transforms.Transform columns differ between the training and the predictive "
                "kernel): unsupported by the B200 solver backend")
        if X_test is None:
            m = self._n
            xt_ptr = None
        else:
            prog, xt = kernel.lower_for(X_test)
            if xt.shape[1] != self._x.shape[1]:
                raise ValueError("X_test must have the same number of input dimensions as the training inputs")
            m = xt.shape[0]
            xt_ptr = _cabi.ptr(xt)
        if diag.shape != (m,):
            raise ValueError("noise diagonal must match the number of test points")
        out = np.empty((m, m))
        self._ctx.check(self._ctx.lib.b200gp_dense_condition(self._h, _cabi.ptr(prog), prog.shape[0], xt_ptr, m,
                                                             _cabi.ptr(diag), _cabi.ptr(out)))
        return ConditionedCovariance.tag(out, True)          # direct.py:88-92: Kss = kernel(X*, X*) + noise
