"""Stationary kernels (reference: src/tinygp/kernels/stationary.py:38-235).

Same constructor signatures and defaults as the reference (``scale`` defaults to 1,
``distance`` defaults to L1 except for ExpSquared which defaults to L2 -- note that
RationalQuadratic therefore uses the *L1* metric by default, stationary.py:56,232-235).
"""

from __future__ import annotations

__all__ = ["Stationary", "Exp", "ExpSquared", "Matern32", "Matern52", "Cosine", "ExpSineSquared",
           "RationalQuadratic"]

import numpy as np

from tinygp_b200.kernels.base import Kernel
from tinygp_b200.kernels.distance import Distance, L1Distance, L2Distance


class Stationary(Kernel):
    opcode: int | None = None
    default_distance = L1Distance
    p1_field: str | None = None     # the field behind program slot p1 (gradient provenance)

    def __init__(self, scale=1.0, distance: Distance | None = None):
        self.scale = scale
        self.distance = self.default_distance() if distance is None else distance

    def _check(self):
        if np.ndim(self.scale):  # stationary.py:77-81
            raise ValueError(
                "Only scalar scales are permitted for stationary kernels; use"
                "transforms.Linear or transforms.Cholesky for more flexiblity"
            )
        if not isinstance(self.distance, Distance) or self.distance.code is None:
            raise NotImplementedError("custom Distance metrics are unsupported by the B200 solver backend")

    def _params(self):
        return float(self.scale), 0.0

    def lower(self, lc):
        self._check()
        p0, p1 = self._params()
        lc.note_leaf(self, "scale", self.p1_field)
        return [(self.opcode, self.distance.code + lc.metric_code(), p0, p1)]


class Exp(Stationary):
    """exp(-r), stationary.py:59-82"""
    opcode = 1


class ExpSquared(Stationary):
    """exp(-r^2 / 2) with r^2 = squared_distance / scale^2, stationary.py:85-106"""
    opcode = 2
    default_distance = L2Distance


class Matern32(Stationary):
    """(1 + sqrt(3) r) exp(-sqrt(3) r), stationary.py:109-129"""
    opcode = 3


class Matern52(Stationary):
    """(1 + sqrt(5) r + 5 r^2 / 3) exp(-sqrt(5) r), stationary.py:132-153"""
    opcode = 4


class Cosine(Stationary):
    """cos(2 pi r), stationary.py:156-175"""
    opcode = 5


class ExpSineSquared(Stationary):
    """exp(-gamma sin^2(pi r)), stationary.py:178-205"""
    opcode = 6
    p1_field = "gamma"

    def __init__(self, scale=1.0, distance: Distance | None = None, gamma=None):
        super().__init__(scale, distance)
        if gamma is None:
            raise ValueError("Missing required argument 'gamma'")
        self.gamma = gamma

    def _params(self):
        return float(self.scale), float(self.gamma)


class RationalQuadratic(Stationary):
    """(1 + r^2 / (2 alpha))^-alpha, stationary.py:208-235"""
    opcode = 7
    p1_field = "alpha"

    def __init__(self, scale=1.0, distance: Distance | None = None, alpha=None):
        super().__init__(scale, distance)
        if alpha is None:
            raise ValueError("Missing required argument 'alpha'")
        self.alpha = alpha

    def _params(self):
        return float(self.scale), float(self.alpha)
