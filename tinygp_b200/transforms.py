"""Input transforms, same names and semantics as ``tinygp.transforms`` (src/tinygp/transforms.py:23-161).

``Linear``, ``Cholesky`` and ``Subspace`` are linear maps of the coordinates, and the stationary kernels they
wrap only see coordinate *differences*, so none of them touches the data: at lowering time they compose into a
small per-leaf matrix ``M`` and the CUDA build kernels measure each leaf's distance on ``M (x1 - x2)``
(include/b200gp.h, B200GP_OP_METRIC).  Different leaves of a sum/product may carry different transforms (e.g. an
additive model over ``Subspace`` kernels).  A general ``Transform(callable, kernel)`` is applied on the host,
point by point like the reference's vmapped ``evaluate``, and its output travels to the device as extra
coordinate columns.
"""

from __future__ import annotations

__all__ = ["Transform", "Linear", "Cholesky", "Subspace"]

from collections.abc import Callable, Sequence
from typing import Any

import numpy as np

from tinygp_b200.kernels.base import Kernel, Lowering


class _Mapped(Kernel):
    """shared lowering: push a matrix on the Lowering state around the wrapped kernel"""

    kernel: Kernel

    def _matrix(self, lc: Lowering) -> np.ndarray:
        raise NotImplementedError

    def _rows(self, owners: list[tuple]) -> list[tuple]:
        """row provenance (Lowering.row_owners) of this node's matrix from that of the matrix it maps"""
        raise NotImplementedError(f"transforms.{type(self).__name__}: log-likelihood gradients cover 0- / 1-D "
                                  "transforms.Linear / Cholesky and Subspace only")

    def lower(self, lc: Lowering):
        prev, prev_owners = lc.matrix, lc.row_owners
        if lc.track:
            lc.row_owners = self._rows(lc.owners())
        lc.matrix = np.atleast_2d(np.asarray(self._matrix(lc), dtype=np.float64))
        try:
            return self.kernel.lower(lc)
        finally:
            lc.matrix, lc.row_owners = prev, prev_owners


def _scaled_rows(node, field: str, kind: str, owners: list[tuple]) -> list[tuple]:
    v = np.asarray(getattr(node, field))
    if v.ndim >= 2:
        return _Mapped._rows(node, owners)
    return [o + ((node, field, r if v.ndim == 1 else 0, kind),) for r, o in enumerate(owners)]


class Transform(_Mapped):
    """transforms.py:23-37 -- ``kernel.evaluate(transform(X1), transform(X2))`` for an arbitrary callable."""

    def __init__(self, transform: Callable[[Any], Any], kernel: Kernel):
        self.transform, self.kernel = transform, kernel

    def _matrix(self, lc):
        pts = lc.coords()
        if lc.matrix is None and lc.scalar_coords:   # 1-D coordinates reach the callable as scalars, as in the reference
            Z = [self.transform(p[0]) for p in pts]
        else:
            Z = [self.transform(p) for p in pts]
        Z = np.asarray(Z, dtype=np.float64).reshape(len(pts), -1)
        return lc.append_columns(Z)


class Linear(_Mapped):
    """transforms.py:40-74 -- ``scale * X`` for 0-/1-D ``scale``, ``scale @ X`` for a matrix."""

    def __init__(self, scale, kernel: Kernel):
        self.scale, self.kernel = scale, kernel

    def _matrix(self, lc):
        cur = lc.current()
        scale = np.asarray(self.scale, dtype=np.float64)
        if scale.ndim < 2:
            return np.broadcast_to(scale, (cur.shape[0],))[:, None] * cur
        if scale.ndim == 2:
            return scale @ cur
        raise ValueError("'scale' must be 0-, 1-, or 2-dimensional")

    def _rows(self, owners):
        return _scaled_rows(self, "scale", "linear", owners)


class Cholesky(_Mapped):
    """transforms.py:77-136 -- ``X / factor`` for 0-/1-D ``factor``, ``solve_triangular(factor, X, lower=True)``
    for a matrix (only its lower triangle is read, as in the reference)."""

    def __init__(self, factor, kernel: Kernel):
        self.factor, self.kernel = factor, kernel

    def _matrix(self, lc):
        cur = lc.current()
        factor = np.asarray(self.factor, dtype=np.float64)
        if factor.ndim < 2:
            return np.broadcast_to(1.0 / factor, (cur.shape[0],))[:, None] * cur
        if factor.ndim == 2:
            L = np.tril(factor)
            if L.shape[0] != L.shape[1] or L.shape[0] != cur.shape[0]:
                raise ValueError("Cholesky factor does not match the input dimension")
            out = np.zeros_like(cur)
            for i in range(L.shape[0]):      # forward substitution (lower=True)
                out[i] = (cur[i] - L[i, :i] @ out[:i]) / L[i, i]
            return out
        raise ValueError("'scale' must be 0-, 1-, or 2-dimensional")

    def _rows(self, owners):
        return _scaled_rows(self, "factor", "cholesky", owners)

    @classmethod
    def from_parameters(cls, diagonal, off_diagonal, kernel: Kernel) -> "Cholesky":
        """transforms.py:108-136"""
        diagonal = np.asarray(diagonal, dtype=np.float64)
        off_diagonal = np.asarray(off_diagonal, dtype=np.float64)
        ndim = diagonal.size
        if off_diagonal.size != ((ndim - 1) * ndim) // 2:
            raise ValueError(
                "Dimension mismatch: expected "
                f"(ndim-1)*ndim/2 = {((ndim - 1) * ndim) // 2} elements in "
                f"'off_diagonal'; got {off_diagonal.size}"
            )
        factor = np.zeros((ndim, ndim))
        factor[np.diag_indices(ndim)] += diagonal
        factor[np.tril_indices(ndim, -1)] += off_diagonal
        return cls(factor, kernel)


class Subspace(_Mapped):
    """transforms.py:139-161 -- ``kernel.evaluate(X1[axis], X2[axis])``."""

    def __init__(self, axis: Sequence[int] | int, kernel: Kernel):
        self.axis, self.kernel = axis, kernel

    def _matrix(self, lc):
        cur = lc.current()
        axis = self.axis if np.ndim(self.axis) == 0 else list(self.axis)
        return cur[axis]

    def _rows(self, owners):
        return [owners[a] for a in np.atleast_1d(self.axis)]
