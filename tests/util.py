"""Shared helpers for the parity tests: map a product kernel expression onto the oracle's classes; build the device
source checks of tests/csrc for the CPU."""

import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest

from oracle import tinygp_np as o
from tinygp_b200 import kernels as K
from tinygp_b200.kernels import quasisep as Q

FP64_RTOL = 5e-7          # the reference's own tolerance (src/tinygp/test_utils.py:9-26)
LOGP_RTOL = 1e-8          # north-star parity target |dlogp| / |logp|


def to_oracle(k):
    if isinstance(k, K.Sum):
        return o.Sum(to_oracle(k.kernel1), to_oracle(k.kernel2))
    if isinstance(k, K.Product):
        return o.Product(to_oracle(k.kernel1), to_oracle(k.kernel2))
    if isinstance(k, K.Constant):
        return o.Constant(k.value)
    if isinstance(k, K.Stationary):
        dist = o.L2Distance() if isinstance(k.distance, K.L2Distance) else o.L1Distance()
        name = type(k).__name__
        cls = getattr(o, name)
        if name == "ExpSineSquared":
            return cls(k.scale, dist, gamma=k.gamma)
        if name == "RationalQuadratic":
            return cls(k.scale, dist, alpha=k.alpha)
        return cls(k.scale, dist)
    if isinstance(k, Q.Sum):
        return o.qs.Sum(to_oracle(k.kernel1), to_oracle(k.kernel2))
    if isinstance(k, Q.Product):
        return o.qs.Product(to_oracle(k.kernel1), to_oracle(k.kernel2))
    if isinstance(k, Q.Scale):
        return o.qs.Scale(to_oracle(k.kernel), k.scale)
    if isinstance(k, Q.CARMA):
        return o.qs.CARMA(k.alpha, k.beta)
    if isinstance(k, Q.Celerite):
        return o.qs.Celerite(k.a, k.b, k.c, k.d)
    if isinstance(k, Q.SHO):
        return o.qs.SHO(k.omega, k.quality, k.sigma)
    if isinstance(k, (Q.Exp, Q.Matern32, Q.Matern52, Q.Cosine)):
        return getattr(o.qs, type(k).__name__)(k.scale, k.sigma)
    raise TypeError(type(k))


def assert_close(a, b, rtol=FP64_RTOL, atol=FP64_RTOL):
    np.testing.assert_allclose(np.asarray(a), np.asarray(b), rtol=rtol, atol=atol)


def rel(a, b):
    return abs(a - b) / abs(b)


def host_library(src, out, deps, flags=()):
    """``src`` (a tests/csrc/*_hostcheck.cu) compiled for the CPU by nvcc into the shared library ``out``, loaded with
    ctypes; rebuilt when ``out`` is older than one of ``deps``.  Skips the calling test when nvcc is not installed."""
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    if not os.path.exists(out) or any(os.path.getmtime(d) > os.path.getmtime(out) for d in deps):
        os.makedirs(os.path.dirname(out), exist_ok=True)
        subprocess.run([nvcc, "-O2", "-std=c++17", "-Wno-deprecated-gpu-targets", *flags, "-Xcompiler", "-fPIC", "-shared",
                        "-o", out, src], check=True)
    return ctypes.CDLL(out)
