"""`jax.random` stand-in: NumPy generators behind key objects.  Streams differ from threefry by construction, so
sample *values* are not reference values — only their statistics are."""

import numpy as _np

from .numpy import _cast


class KeyArray:
    def __init__(self, seed):
        self.seed = seed

    def _rng(self):
        return _np.random.default_rng(self.seed)


def PRNGKey(seed):
    return KeyArray([int(seed)])


key = PRNGKey


def split(k, num=2):
    return [KeyArray(list(k.seed) + [i]) for i in range(num)]


def normal(k, shape=(), dtype=float):
    return _cast(k._rng().standard_normal(shape).astype(dtype))


def uniform(k, shape=(), dtype=float, minval=0.0, maxval=1.0):
    return _cast(k._rng().uniform(minval, maxval, shape).astype(dtype))
