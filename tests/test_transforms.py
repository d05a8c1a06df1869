"""Input transforms (reference: src/tinygp/transforms.py:23-161, docs in transforms.py:44-55,
81-92,143-154).  CPU tests check the host lowering (per-leaf metric matrices, augmented columns) through a
Python restatement of the device interpreter; GPU tests check the CUDA build kernels and the full
GaussianProcess path against the oracle, which maps the *points* like the reference does."""

import numpy as np
import pytest

from oracle import tinygp_np as ref
from tinygp_b200 import kernels, transforms
from tinygp_b200.kernels.base import OP_METRIC

RTOL = 1e-12


def _interp(prog, x1, x2):
    """Python restatement of kprog_eval (csrc/dense.cu) for ONE pair of (device) coordinates."""
    rows = [tuple(r) for r in prog]
    metrics = []
    i = 0
    while int(rows[i][0]) == OP_METRIC:
        _, mid, r, c = rows[i]
        r, c = int(r), int(c)
        assert int(mid) == len(metrics) + 1 and c == len(x1)
        nd = -(-r * c // 4)
        flat = np.array(rows[i + 1:i + 1 + nd]).ravel()[:r * c]
        metrics.append(flat.reshape(r, c))
        i += 1 + nd
    d = np.asarray(x1, float) - np.asarray(x2, float)
    st = []
    for op, dcode, p0, p1 in rows[i:]:
        op, dcode = int(op), int(dcode)
        if op == 16:
            b = st.pop(); st[-1] = st[-1] + b; continue
        if op == 17:
            b = st.pop(); st[-1] = st[-1] * b; continue
        if op == 0:
            st.append(p0); continue
        z = d if dcode >> 1 == 0 else metrics[(dcode >> 1) - 1] @ d
        l1, l2sq = np.abs(z).sum(), (z * z).sum()
        l2 = dcode & 1
        if op in (2, 7):
            r2 = (l2sq if l2 else l1 * l1) / (p0 * p0)
            st.append(np.exp(-0.5 * r2) if op == 2 else (1 + 0.5 * r2 / p1) ** (-p1))
            continue
        dist = (l1 if l2sq == 0 else np.sqrt(l2sq)) if l2 else l1
        if op in (8, 9):
            st.append(np.exp(-p0 * dist) * (np.cos(p1 * dist) if op == 8 else np.sin(p1 * dist)))
            continue
        r = dist / p0
        if op == 1:
            v = np.exp(-r)
        elif op == 3:
            v = (1 + np.sqrt(3) * r) * np.exp(-np.sqrt(3) * r)
        elif op == 4:
            a = np.sqrt(5) * r
            v = (1 + a + a * a / 3) * np.exp(-a)
        elif op == 5:
            v = np.cos(2 * np.pi * r)
        else:
            v = np.exp(-p1 * np.sin(np.pi * r) ** 2)
        st.append(v)
    assert len(st) == 1
    return st[0]


def _L(d, seed=3):
    rng = np.random.default_rng(seed)
    return np.tril(rng.normal(size=(d, d)) * 0.3) + np.diag(rng.uniform(0.7, 1.5, d))


def _warp(x):   # a non-linear map R^3 -> R^2
    return np.array([np.sin(x[0]) + x[1] ** 2, np.tanh(x[2]) - x[0]])


def _cases():
    """name, our kernel, oracle kernel, ndim"""
    S = np.random.default_rng(0).normal(size=(2, 3))
    L3 = _L(3)
    K, R, T, RT = kernels, ref, transforms, ref
    l2 = lambda: (K.L2Distance(), R.L2Distance())  # noqa: E731
    out = []
    out.append(("linear_scalar", T.Linear(1 / 4.5, K.Matern32()), RT.Linear(1 / 4.5, R.Matern32()), 1))
    out.append(("cholesky_scalar", T.Cholesky(4.5, K.Matern32()), RT.Cholesky(4.5, R.Matern32()), 1))
    out.append(("linear_vec", T.Linear([0.5, 2.0, 1.5], K.ExpSquared()), RT.Linear([0.5, 2.0, 1.5], R.ExpSquared()), 3))
    a, b = l2()
    out.append(("linear_mat", T.Linear(S, K.Matern52(1.3, distance=a)), RT.Linear(S, R.Matern52(1.3, distance=b)), 3))
    out.append(("cholesky_vec", T.Cholesky([0.5, 2.0, 1.5], K.ExpSquared()), RT.Cholesky([0.5, 2.0, 1.5], R.ExpSquared()), 3))
    out.append(("cholesky_mat", 1.7 * T.Cholesky(L3, K.ExpSquared()), 1.7 * RT.Cholesky(L3, R.ExpSquared()), 3))
    out.append(("cholesky_params",
                T.Cholesky.from_parameters([1.0, 2.0, 0.7], [0.1, -0.2, 0.3], K.ExpSquared(0.9)),
                RT.Cholesky.from_parameters([1.0, 2.0, 0.7], [0.1, -0.2, 0.3], R.ExpSquared(0.9)), 3))
    out.append(("subspace_int", T.Subspace(1, K.Matern32()), RT.Subspace(1, R.Matern32()), 3))
    out.append(("subspace_tuple", T.Subspace((0, 2), K.ExpSquared(0.8)), RT.Subspace((0, 2), R.ExpSquared(0.8)), 3))
    # an additive model: every leaf has its own transform, one leaf has none
    out.append(("additive",
                T.Subspace(0, K.Matern32(0.9)) + 0.5 * T.Subspace((1, 2), K.ExpSquared(1.1)) + 0.3 * K.ExpSquared(2.0),
                RT.Subspace(0, R.Matern32(0.9)) + 0.5 * RT.Subspace((1, 2), R.ExpSquared(1.1)) + 0.3 * R.ExpSquared(2.0),
                3))
    # nesting composes:  Linear(S) then Subspace(1) of the 2-D image
    out.append(("nested", T.Linear(S, T.Subspace(1, K.Exp(0.7))), RT.Linear(S, RT.Subspace(1, R.Exp(0.7))), 3))
    out.append(("nested_chol", T.Cholesky(L3, T.Linear([1.0, 0.5, 2.0], K.ExpSquared())),
                RT.Cholesky(L3, RT.Linear([1.0, 0.5, 2.0], R.ExpSquared())), 3))
    # general callables: host-computed columns; the sibling leaf must not see them
    out.append(("callable", T.Transform(_warp, K.ExpSquared(0.8)) + 0.2 * K.ExpSquared(1.5),
                RT.Transform(_warp, R.ExpSquared(0.8)) + 0.2 * R.ExpSquared(1.5), 3))
    out.append(("callable_scalar", T.Transform(np.log, K.Matern32(0.5)), RT.Transform(np.log, R.Matern32(0.5)), 0))
    out.append(("callable_nested", T.Linear([0.5, 1.0, 2.0], T.Transform(_warp, T.Subspace(1, K.Exp()))),
                RT.Linear([0.5, 1.0, 2.0], RT.Transform(_warp, RT.Subspace(1, R.Exp()))), 3))
    return out


CASES = _cases()


def _points(nd, n, seed):
    rng = np.random.default_rng(seed)
    if nd == 0:
        return rng.uniform(0.5, 3.0, n)          # 1-D coordinates given as shape (N,), positive for log
    return rng.normal(size=(n, nd))


@pytest.mark.parametrize("name,k,kr,nd", CASES, ids=[c[0] for c in CASES])
def test_lowering_matches_point_transform(name, k, kr, nd):
    X1, X2 = _points(nd, 7, 1), _points(nd, 5, 2)
    prog1, x1 = k.lower_for(X1)
    prog2, x2 = k.lower_for(X2)
    assert np.array_equal(prog1, prog2)           # the program does not depend on the data
    want = kr(X1, X2)
    got = np.array([[_interp(prog1, a, b) for b in x2] for a in x1])
    np.testing.assert_allclose(got, want, rtol=RTOL, atol=1e-14)


def test_reference_docstring_identities_oracle():
    """transforms.py:47-55, 84-92, 146-154"""
    k0 = ref.Matern32(4.5)
    for k1 in (ref.Linear(1.0 / 4.5, ref.Matern32()), ref.Cholesky(4.5, ref.Matern32())):
        np.testing.assert_allclose(k0(np.array([0.5]), np.array([0.1])), k1(np.array([0.5]), np.array([0.1])))
    k = ref.Subspace(1, ref.Matern32())
    np.testing.assert_allclose(k(np.array([[0.5, 0.1]]), np.array([[-0.4, 0.7]])),
                               k(np.array([[100.5, 0.1]]), np.array([[-70.4, 0.7]])))


def test_program_layout_and_limits():
    k = transforms.Subspace(1, kernels.Matern32()) + kernels.Exp()
    with pytest.raises(ValueError):
        k.program()                                # needs coordinates
    prog, x = k.lower_for(np.zeros((4, 3)))
    assert x.shape == (4, 3)
    assert prog[0].tolist() == [OP_METRIC, 1, 1, 3] and prog[1].tolist() == [0, 1, 0, 0]
    assert prog[2].tolist()[:2] == [3, 2] and prog[3].tolist()[:2] == [1, 0] and prog[4][0] == 16
    # identical transforms share one metric
    k2 = transforms.Linear(2.0, kernels.Exp()) + transforms.Linear(2.0, kernels.Matern32())
    prog, _ = k2.lower_for(np.zeros((4, 2)))
    assert int((prog[:, 0] == OP_METRIC).sum()) == 1
    # at most three distinct transforms, at most 8 dimensions
    k4 = sum(transforms.Subspace(i, kernels.Exp()) for i in range(4))
    with pytest.raises(NotImplementedError):
        k4.lower_for(np.zeros((4, 4)))
    with pytest.raises(NotImplementedError):
        transforms.Linear(2.0, kernels.Exp()).lower_for(np.zeros((4, 9)))
    with pytest.raises(ValueError):
        transforms.Linear(np.ones((2, 2, 2)), kernels.Exp()).lower_for(np.zeros((4, 2)))
    with pytest.raises(ValueError):
        transforms.Cholesky.from_parameters(np.ones(3), np.ones(2), kernels.Exp())
    # untransformed kernels keep their old programs and coordinates
    X = np.random.default_rng(0).normal(size=(5, 2))
    prog, x = (1.5 * kernels.ExpSquared(2.0)).lower_for(X)
    assert np.array_equal(prog, (1.5 * kernels.ExpSquared(2.0)).program()) and np.array_equal(x, X)


# ------------------------------------------------------------------------------------------------
# GPU parity
# ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name,k,kr,nd", CASES, ids=[c[0] for c in CASES])
def test_kernel_matrix_gpu(name, k, kr, nd):
    X1, X2 = _points(nd, 150, 1), _points(nd, 70, 2)
    np.testing.assert_allclose(k(X1, X2), kr(X1, X2), rtol=RTOL, atol=1e-14)
    np.testing.assert_allclose(k(X1), kr(X1), rtol=RTOL, atol=1e-14)
    y = np.random.default_rng(5).normal(size=70)
    np.testing.assert_allclose(k.matmul(X1, X2, y), kr(X1, X2) @ y, rtol=1e-11, atol=1e-12)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["cholesky_mat", "additive", "callable", "linear_mat"])
def test_gp_with_transforms_gpu(name):
    import tinygp_b200 as tg
    _, k, kr, nd = next(c for c in CASES if c[0] == name)
    n = 700
    X, Xt = _points(nd, n, 11), _points(nd, 40, 12)
    y = np.sin(X.sum(axis=-1) if nd else X)
    gp = tg.GaussianProcess(k, X, diag=0.05)
    gpr = ref.GaussianProcess(kr, X, diag=0.05)
    lp, lpr = gp.log_probability(y), gpr.log_probability(y)
    assert abs(lp - lpr) / abs(lpr) < 1e-8          # north_star tolerance
    mu, var = gp.predict(y, Xt, return_var=True)
    mur, varr = gpr.predict(y, Xt, return_var=True)
    np.testing.assert_allclose(mu, mur, rtol=1e-7, atol=1e-9)
    np.testing.assert_allclose(var, varr, rtol=1e-6, atol=1e-9)


@pytest.mark.gpu
def test_transforms_int8_path_gpu():
    """the int8 fixed-point factorisation sees the same build kernel: force it at a small size"""
    import tinygp_b200 as tg
    from tinygp_b200 import _cabi
    _, k, kr, nd = next(c for c in CASES if c[0] == "cholesky_mat")
    ctx = _cabi.get_context()
    X = _points(nd, 1536, 21)
    y = np.cos(X.sum(axis=-1))
    want = ref.GaussianProcess(kr, X, diag=0.1).log_probability(y)
    ctx.set_option("ozaki_min_n", 0)
    ctx.set_option("nb", 256)
    try:
        got = tg.GaussianProcess(k, X, diag=0.1).log_probability(y)
    finally:
        ctx.set_option("ozaki_min_n", 8192)
        ctx.set_option("nb", 1024)
    assert abs(got - want) / abs(want) < 1e-8


@pytest.mark.gpu
def test_bad_metric_programs_rejected_gpu():
    from tinygp_b200 import _cabi
    ctx = _cabi.get_context()
    X = np.zeros((4, 2))
    out = np.empty((4, 4))

    def call(prog, nd=2):
        prog = np.ascontiguousarray(np.array(prog, dtype=np.float64))
        return ctx.lib.b200gp_kernel_matrix(ctx.handle, _cabi.ptr(prog), prog.shape[0], _cabi.ptr(X), 4,
                                            _cabi.ptr(X), 4, nd, _cabi.ptr(out))

    good = [[OP_METRIC, 1, 1, 2], [1, 0, 0, 0], [1, 2, 1.0, 0]]
    assert call(good) == 0
    assert call([[OP_METRIC, 2, 1, 2], [1, 0, 0, 0], [1, 2, 1.0, 0]]) != 0      # ids must start at 1
    assert call([[OP_METRIC, 1, 1, 3], [1, 0, 0, 0], [1, 2, 1.0, 0]]) != 0      # width != ndim
    assert call([[OP_METRIC, 1, 3, 2], [1, 0, 0, 0], [1, 2, 1.0, 0]]) != 0      # truncated definition
    assert call([[1, 2, 1.0, 0]]) != 0                                            # undefined metric
    assert call([[OP_METRIC, 1, 1, 2], [np.nan, 0, 0, 0], [1, 2, 1.0, 0]]) != 0  # non-finite matrix
