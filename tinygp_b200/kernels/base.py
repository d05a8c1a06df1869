"""Kernel expression surface (reference: src/tinygp/kernels/base.py).

A kernel here is a plain parameter holder.  ``Kernel.__call__`` (base.py:84-103)
does not vmap a Python ``evaluate``; it lowers the expression to a postfix *kernel
program* (include/b200gp.h) and runs the pairwise-build CUDA kernel.
"""

from __future__ import annotations

__all__ = ["Kernel", "Conditioned", "Custom", "Sum", "Product", "Constant", "DotProduct", "Polynomial", "Lowering"]

import numpy as np

from tinygp_b200 import _cabi

OP_CONST, OP_ADD, OP_MUL, OP_METRIC = 0, 16, 17, 32


def _as_coords(X):
    X = np.asarray(X, dtype=np.float64)
    if X.ndim == 1:
        return np.ascontiguousarray(X[:, None]), True
    if X.ndim == 2:
        return np.ascontiguousarray(X), False
    raise ValueError("coordinates must have shape (N,) or (N, D); pytrees are not supported by the B200 backend")


class Lowering:
    """State threaded through ``Kernel.lower``: the input transform in force at the current node.

    The device interpreter evaluates a stationary leaf on ``M (x1 - x2)`` for a per-leaf matrix ``M``
    (include/b200gp.h, B200GP_OP_METRIC).  ``transforms.Linear/Cholesky/Subspace`` (transforms.py:57-161)
    compose into ``M`` directly.  A general ``transforms.Transform(callable)`` (transforms.py:23-37) is
    applied on the host, point by point, and its output is appended to the coordinates as extra columns
    which the leaf's matrix then selects -- so a program is always lowered *for* a coordinate array and the
    (possibly augmented) coordinates are what goes to the device.
    """

    MAX_METRICS = 3
    MAX_DIM = 8

    def __init__(self, X=None, scalar_coords=False, track=False):
        self.X = X                    # (N, D) or None when lowering without coordinates
        self.ndim0 = None if X is None else X.shape[1]   # width before any host-computed columns are appended
        self.scalar_coords = scalar_coords
        self.matrix = None            # None = untransformed coordinates
        self.metrics: list[np.ndarray] = []
        # slot provenance, recorded when `track` is set (Kernel.lower_for_grad):
        #   leaf_params[k] = (node, p0 field, p1 field or None) of the k-th leaf / CONST instruction, in program order;
        #   row_owners[r] = the (node, field, index, kind) row scalings that make row r of the current matrix, kind
        #   "linear" (row scaled by node.field[index]) or "cholesky" (scaled by 1 / node.field[index]);
        #   metric_owners[m] = row_owners of metric m.  Metrics are shared only between leaves with the same owners.
        self.track = track
        self.leaf_params: list[tuple] = []
        self.row_owners: list[tuple] | None = None
        self.metric_owners: list[list[tuple]] = []

    # -- used by transform nodes ----------------------------------------------------------
    def width(self) -> int:
        if self.X is None:
            raise ValueError("a kernel with input transforms can only be lowered for given coordinates "
                             "(use Kernel.lower_for(X))")
        return self.X.shape[1]

    def owners(self) -> list[tuple]:
        return [()] * self.current().shape[0] if self.row_owners is None else self.row_owners

    def current(self) -> np.ndarray:
        return np.eye(self.ndim0, self.width()) if self.matrix is None else self.matrix

    def coords(self) -> np.ndarray:
        """coordinates seen by the current node, one row per point"""
        self.width()
        if self.matrix is None:
            return self.X[:, :self.ndim0]
        return self.X[:, :self.matrix.shape[1]] @ self.matrix.T   # columns appended later are not seen

    def append_columns(self, Z: np.ndarray) -> np.ndarray:
        """augment the coordinates with host-computed columns; returns the matrix selecting them"""
        w0 = self.width()
        self.X = np.ascontiguousarray(np.concatenate([self.X, Z], axis=1))
        sel = np.zeros((Z.shape[1], self.X.shape[1]))
        sel[np.arange(Z.shape[1]), w0 + np.arange(Z.shape[1])] = 1.0
        if self.matrix is not None:  # the enclosing matrix refers to the old, narrower coordinates
            self.matrix = np.pad(self.matrix, ((0, 0), (0, Z.shape[1])))
        return sel

    # -- used by leaves -------------------------------------------------------------------
    def note_leaf(self, node, p0_field: str, p1_field: str | None = None):
        if self.track:
            self.leaf_params.append((node, p0_field, p1_field))

    def metric_code(self) -> int:
        if self.matrix is None:
            return 0
        M = np.asarray(self.matrix, dtype=np.float64)
        owners = self.owners() if self.track else None
        for i, other in enumerate(self.metrics):
            k = min(other.shape[1], M.shape[1])
            if other.shape[0] == M.shape[0] and np.array_equal(other[:, :k], M[:, :k]) \
                    and not other[:, k:].any() and not M[:, k:].any() \
                    and (not self.track or self.metric_owners[i] == owners):
                return 2 * (i + 1)
        if len(self.metrics) == self.MAX_METRICS:
            raise NotImplementedError(f"at most {self.MAX_METRICS} distinct input transforms per kernel expression")
        self.metrics.append(M.copy())
        if self.track:
            self.metric_owners.append(owners)
        return 2 * len(self.metrics)

    def metric_rows(self) -> list[tuple[float, float, float, float]]:
        rows: list[tuple[float, float, float, float]] = []
        if not self.metrics:
            return rows
        w = self.width()
        for i, M in enumerate(self.metrics):
            M = np.pad(M, ((0, 0), (0, w - M.shape[1])))
            if M.shape[0] > self.MAX_DIM or w > self.MAX_DIM:
                raise NotImplementedError(f"transformed kernels support at most {self.MAX_DIM} (augmented) input "
                                          "dimensions on the B200 backend")
            if not np.all(np.isfinite(M)):
                raise ValueError("non-finite input transform")
            rows.append((float(OP_METRIC), float(i + 1), float(M.shape[0]), float(w)))
            flat = np.zeros(-(-M.size // 4) * 4)
            flat[:M.size] = M.ravel()
            rows.extend(tuple(r) for r in flat.reshape(-1, 4))
        return rows


class Kernel:
    """Base class (base.py:29-126)."""

    # `ndarray * kernel` must reach Kernel.__rmul__ (as a jax array does, returning NotImplemented) instead of
    # broadcasting into an object array; the non-scalar Constant it builds then fails in evaluate (base.py:203-209)
    __array_ufunc__ = None

    def lower(self, lc: Lowering) -> list[tuple[int, int, float, float]]:
        raise NotImplementedError(
            f"{type(self).__name__} cannot be lowered to a device kernel program: "
            "unsupported by the B200 solver backend (only stationary kernels, their sums/products and "
            "input transforms of them)"
        )

    def program(self) -> np.ndarray:
        """the kernel program of an expression without input transforms"""
        lc = Lowering()
        instr = self.lower(lc)
        return np.ascontiguousarray(np.array(instr, dtype=np.float64).reshape(-1, _cabi.PROG_STRIDE))

    def lower_for(self, X) -> tuple[np.ndarray, np.ndarray]:
        """(program, device coordinates) for the coordinates X; the coordinates are X itself unless the
        expression holds a general ``transforms.Transform``, whose output is appended as extra columns."""
        x, scalar = _as_coords(X)
        lc = Lowering(x, scalar)
        instr = self.lower(lc)
        if lc.X.shape[1] != lc.ndim0:
            # columns were appended: leaves on the untransformed coordinates must not see them
            lc.matrix = np.eye(lc.ndim0, lc.X.shape[1])
            instr = [(op, d + lc.metric_code(), p0, p1) if (0 < op < OP_ADD and d < 2) else (op, d, p0, p1)
                     for (op, d, p0, p1) in instr]
        rows = lc.metric_rows() + instr
        prog = np.ascontiguousarray(np.array(rows, dtype=np.float64).reshape(-1, _cabi.PROG_STRIDE))
        return prog, np.ascontiguousarray(lc.X)

    def lower_for_grad(self, X) -> tuple[np.ndarray, np.ndarray, list[tuple], list[list[tuple]]]:
        """``lower_for(X)`` with slot provenance: (program, coordinates, leaf_params, metric_owners) as recorded in
        ``Lowering``.  Raises NotImplementedError for expressions without device gradients."""
        x, scalar = _as_coords(X)
        lc = Lowering(x, scalar, track=True)
        instr = self.lower(lc)
        if sum(1 for op, *_ in instr if op not in (OP_ADD, OP_MUL)) != len(lc.leaf_params):
            raise NotImplementedError(
                f"{type(self).__name__}: log-likelihood gradients cover stationary kernels, Constant, their sums and "
                "products and 0- / 1-D transforms.Linear / Cholesky and Subspace; this expression holds a kernel without "
                "a differentiable device program (e.g. a quasiseparable kernel evaluated densely)")
        prog = np.ascontiguousarray(np.array(lc.metric_rows() + instr, dtype=np.float64).reshape(-1, _cabi.PROG_STRIDE))
        return prog, np.ascontiguousarray(lc.X), lc.leaf_params, lc.metric_owners

    # -- evaluation ---------------------------------------------------------------------
    def evaluate(self, X1, X2):
        """Scalar evaluation at a single pair of coordinates (base.py:37-56)."""
        x1 = np.atleast_1d(np.asarray(X1, dtype=np.float64))[None, :]
        x2 = np.atleast_1d(np.asarray(X2, dtype=np.float64))[None, :]
        return self(x1, x2)[0, 0]

    def evaluate_diag(self, X):
        return self.evaluate(X, X)

    def __call__(self, X1, X2=None):
        ctx = _cabi.get_context()
        prog, x1 = self.lower_for(X1)
        if X2 is None:  # base.py:85-93
            out = np.empty(x1.shape[0])
            ctx.check(ctx.lib.b200gp_kernel_diag(ctx.handle, _cabi.ptr(prog), prog.shape[0], _cabi.ptr(x1),
                                                 x1.shape[0], x1.shape[1], _cabi.ptr(out)))
            return out
        _, x2 = self.lower_for(X2)
        if x1.shape[1] != x2.shape[1]:
            raise ValueError("X1 and X2 must have the same number of input dimensions")
        out = np.empty((x1.shape[0], x2.shape[0]))
        ctx.check(ctx.lib.b200gp_kernel_matrix(ctx.handle, _cabi.ptr(prog), prog.shape[0], _cabi.ptr(x1), x1.shape[0],
                                               _cabi.ptr(x2), x2.shape[0], x1.shape[1], _cabi.ptr(out)))
        return out

    def matmul(self, X1, X2=None, y=None):
        """base.py:68-82 -- k(X1, X2) @ y without materialising K for vector y."""
        if y is None:
            assert X2 is not None
            y = X2
            X2 = None
        if X2 is None:
            X2 = X1
        y = np.asarray(y, dtype=np.float64)
        ctx = _cabi.get_context()
        prog, x1 = self.lower_for(X1)
        _, x2 = self.lower_for(X2)
        if x1.shape[1] != x2.shape[1]:
            raise ValueError("X1 and X2 must have the same number of input dimensions")
        if y.shape[0] != x2.shape[0]:
            raise ValueError("dimension mismatch")
        cols = np.ascontiguousarray(y.reshape(x2.shape[0], -1).T)   # one device matvec per right-hand side
        out = np.empty((cols.shape[0], x1.shape[0]))
        for r in range(cols.shape[0]):
            ctx.check(ctx.lib.b200gp_kernel_matvec(ctx.handle, _cabi.ptr(prog), prog.shape[0], _cabi.ptr(x1),
                                                   x1.shape[0], _cabi.ptr(x2), x2.shape[0], x1.shape[1],
                                                   _cabi.ptr(cols[r]), _cabi.ptr(out[r])))
        return np.ascontiguousarray(out.T).reshape((x1.shape[0],) + y.shape[1:])

    # -- algebra (base.py:105-126) --------------------------------------------------------
    def __add__(self, other):
        if isinstance(other, Kernel):
            return Sum(self, other)
        return Sum(self, Constant(other))

    def __radd__(self, other):
        if not isinstance(other, Kernel) and np.ndim(other) == 0 and other == 0:
            return self
        if isinstance(other, Kernel):
            return Sum(other, self)
        return Sum(Constant(other), self)

    def __mul__(self, other):
        if isinstance(other, Kernel):
            return Product(self, other)
        return Product(self, Constant(other))

    def __rmul__(self, other):
        if isinstance(other, Kernel):
            return Product(other, self)
        return Product(Constant(other), self)


class Sum(Kernel):
    """base.py:170-177"""

    def __init__(self, kernel1: Kernel, kernel2: Kernel):
        self.kernel1, self.kernel2 = kernel1, kernel2

    def lower(self, lc):
        return self.kernel1.lower(lc) + self.kernel2.lower(lc) + [(OP_ADD, 0, 0.0, 0.0)]


class Product(Kernel):
    """base.py:180-187"""

    def __init__(self, kernel1: Kernel, kernel2: Kernel):
        self.kernel1, self.kernel2 = kernel1, kernel2

    def lower(self, lc):
        return self.kernel1.lower(lc) + self.kernel2.lower(lc) + [(OP_MUL, 0, 0.0, 0.0)]


class Constant(Kernel):
    """base.py:190-209"""

    def __init__(self, value):
        if np.ndim(value) != 0:
            raise ValueError("The value of a constant kernel must be a scalar")
        self.value = float(value)

    def lower(self, lc):
        lc.note_leaf(self, "value")
        return [(OP_CONST, 0, self.value, 0.0)]


class Conditioned(Kernel):
    """The covariance of a process conditioned on data (base.py:129-153), evaluated matrix-wise:
    k*(X1, X2) - [L^-1 k(X, X1)]^T [L^-1 k(X, X2)]."""

    def __init__(self, X, solver, kernel: Kernel):
        self.X, self.solver, self.kernel = X, solver, kernel

    def __call__(self, X1, X2=None):
        if X2 is None:
            K = self.solver.solve_triangular(self.kernel(self.X, X1))
            return self.kernel(X1) - np.sum(K * K, axis=0)
        # the rectangular block of the joint conditioned covariance of [X1; X2]: kernel values from the build kernel, one
        # triangular solve, and Kss - A^T A by the device GEMM (b200gp_gram_downdate) -- no host matrix product
        X1, X2 = np.asarray(X1, dtype=np.float64), np.asarray(X2, dtype=np.float64)
        m1 = X1.shape[0]
        XX = np.concatenate((X1, X2), axis=0)
        At = np.ascontiguousarray(self.solver.solve_triangular(self.kernel(self.X, XX)).T)
        C = np.ascontiguousarray(self.kernel(XX, XX))
        ctx = _cabi.get_context()
        ctx.check(ctx.lib.b200gp_gram_downdate(ctx.handle, _cabi.ptr(At), At.shape[0], At.shape[1], _cabi.ptr(C)))
        return C[:m1, m1:]

    def matmul(self, X1, X2=None, y=None):
        if y is None:
            y, X2 = X2, None
        if X2 is None:
            X2 = X1
        return self(X1, X2) @ np.asarray(y, dtype=np.float64)


class Custom(Kernel):
    """base.py:156-167 -- arbitrary Python callables cannot run inside the CUDA build kernel."""

    def __init__(self, function):
        self.function = function


class DotProduct(Kernel):
    """base.py:212-225 -- non-stationary: out of scope of the B200 backend (lower() raises)."""


class Polynomial(Kernel):
    """base.py:228-249 -- non-stationary: out of scope of the B200 backend (lower() raises)."""

    def __init__(self, order, scale=1.0, sigma=0.0):
        self.order, self.scale, self.sigma = order, scale, sigma
