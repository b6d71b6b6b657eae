"""The CGLB oracle (tests/cglb_oracle.py) on the reference's four tests (tests/gpflow/models/test_cglb.py, the same
RandomState(999) data), against dense algebra, and its P > 1 refusal; the parameter-gradient oracle
(tests/cglb_grad_oracle.py) against the dense adjoints and against central differences of the bound."""
import numpy as np
import pytest
from scipy.linalg import solve_triangular

from oracle import gp_oracle as O
from tests import cglb_grad_oracle as CG
from tests import cglb_oracle as C
from tests import kernel_grad_oracle as KG


def _data(rng):
    n, t, d = 100, 20, 2
    x = rng.randn(n, d)
    xs = rng.randn(t, d)
    c = np.array([[-1.4], [0.5]])
    y = np.sin(x @ c + 0.5 * rng.randn(n, 1))
    z = rng.randn(10, 2)
    return (x, y), z, xs


def _sgpr_terms(x, y, z, k, s, jitter=1e-6):
    """sgpr.py:214-271: (logdet_term, quad_term)."""
    N = x.shape[0]
    L, A, LB, AAT = C.common(x, z, k, s, jitter)
    trace_k = np.sum(k.K_diag(x)) / s
    logdet = -(np.sum(np.log(np.diag(LB))) + 0.5 * N * np.log(s) + 0.5 * (trace_k - np.trace(AAT)))
    c = solve_triangular(LB, A @ y, lower=True) / np.sqrt(s)
    quad = -0.5 * (np.sum(y ** 2) / s - np.sum(c ** 2))
    return logdet, quad


def test_cglb_check_basics():
    (x, y), z, _ = _data(np.random.RandomState(999))
    k, s = O.SquaredExponential(), 0.2
    b = C.bound(x, y, z, k, s, np.zeros((1, x.shape[0])))
    sgpr_logdet, sgpr_quad = _sgpr_terms(x, y, z, k, s)
    np.testing.assert_almost_equal(sgpr_quad, b["quad"])
    assert b["logdet"] >= sgpr_logdet
    assert b["logdet"] <= -0.5 * np.linalg.slogdet(k.K(x) + s * np.eye(x.shape[0]))[1]


def test_conjugate_gradient_convergence():
    (x, y), z, _ = _data(np.random.RandomState(999))
    k, s = O.SquaredExponential(), 1e-3
    K = k.K(x) + s * np.eye(x.shape[0])
    _, A, LB, _ = C.common(x, z, k, s)
    v, _, _ = C.conjugate_gradient(K, y.T, np.zeros_like(y.T), A, LB, s, 0.01, 200, 200)
    np.testing.assert_allclose(np.linalg.solve(K, y), v.T, rtol=0.1)


def test_cglb_quad_term_guarantees():
    (x, y), z, _ = _data(np.random.RandomState(999))
    k, s, max_error = O.SquaredExponential(), 1e-2, 1e-2
    K = k.K(x) + s * np.eye(x.shape[0])
    chol_quad = -0.5 * np.sum(solve_triangular(np.linalg.cholesky(K), y, lower=True) ** 2)
    v, _, _ = C.run_cg(x, y, z, k, s, np.zeros((1, x.shape[0])), max_error, 100, 10)
    q = C.bound(x, y, z, k, s, v)["quad"]
    assert q <= chol_quad
    assert abs(q - chol_quad) <= max_error


def test_cglb_predict():
    (x, y), z, xs = _data(np.random.RandomState(999))
    k, s = O.SquaredExponential(), 0.2
    N = x.shape[0]
    K = k.K(x) + s * np.eye(N)
    gpr_mean = k.K(xs, x) @ np.linalg.solve(K, y)
    L, A, LB, _ = C.common(x, z, k, s)
    c = solve_triangular(LB, A @ y, lower=True) / np.sqrt(s)
    tmp1 = solve_triangular(L, k.K(z, xs), lower=True)
    tmp2 = solve_triangular(LB, tmp1, lower=True)
    sgpr_mean = tmp2.T @ c
    sgpr_var = k.K_diag(xs) + np.sum(tmp2 ** 2, 0) - np.sum(tmp1 ** 2, 0)
    v0 = np.zeros((1, N))
    v, _, _ = C.run_cg(x, y, z, k, s, v0, 1e6, 100, 40)
    mean, var = C.predict_f(x, y, z, k, s, v, xs)
    assert np.allclose(sgpr_mean, mean) and np.allclose(sgpr_var[:, None], var)
    v, _, _ = C.run_cg(x, y, z, k, s, v0, 1e-12, 100, 40)
    mean, _ = C.predict_f(x, y, z, k, s, v, xs)
    assert np.allclose(gpr_mean, mean)


def test_bound_below_exact_lml():
    (x, y), z, _ = _data(np.random.RandomState(999))
    k, s = O.Matern52(), 0.1
    N = x.shape[0]
    K = k.K(x) + s * np.eye(N)
    lml = -0.5 * (N * C.LOG2PI + np.linalg.slogdet(K)[1] + (y.T @ np.linalg.solve(K, y)).item())
    v, _, _ = C.run_cg(x, y, z, k, s, np.zeros((1, N)), 1e-2, 100, 40)
    assert C.bound(x, y, z, k, s, v)["elbo"] <= lml
    # at v = K^-1 y the quadratic term is exact
    b = C.bound(x, y, z, k, s, np.linalg.solve(K, y).T)
    np.testing.assert_allclose(b["quad"], -0.5 * (y.T @ np.linalg.solve(K, y)).item(), rtol=1e-9)


def test_cg_refuses_several_outputs():
    (x, y), z, _ = _data(np.random.RandomState(999))
    y2 = np.hstack([y, 2 * y])
    with pytest.raises(ValueError, match="broadcast"):
        C.run_cg(x, y2, z, O.SquaredExponential(), 0.2, np.zeros((2, x.shape[0])), 1e-3, 10, 5)


def test_adjoints_against_finite_differences():
    """Every closed form of the gradient against central differences of the bound in its input matrices (K^ and Kuu
    perturbed symmetrically), with s entering both K^ = K + s I and the Nystrom terms."""
    rng = np.random.default_rng(4)
    N, M, D, P = 40, 6, 2, 2
    X, Z = rng.standard_normal((N, D)), rng.standard_normal((M, D))
    k = O.Matern52(variance=1.3, lengthscales=0.9)
    s = 0.4
    K, Kuf, Kuu = k.K(X), k.K(Z, X), k.K(Z) + 1e-6 * np.eye(M)
    kd = k.K_diag(X)
    e = rng.standard_normal((N, P))
    v = 0.3 * rng.standard_normal((P, N))
    adj = C.bound_adjoints(K + s * np.eye(N), Kuf, Kuu, kd, s, e, v)
    f = lambda **kw: C.bound_from(**{**dict(Kh=K + s * np.eye(N), Kuf=Kuf, Kuu=Kuu, kdiag=kd, s=s, e=e, v=v), **kw})
    h = 1e-6

    def sym_fd(name, A, i, j):
        E = np.zeros_like(A)
        E[i, j] += h
        E[j, i] += h if i != j else 0.0
        return (f(**{name: A + E}) - f(**{name: A - E})) / (2 * h)

    for (i, j) in [(0, 0), (3, 1), (17, 9), (39, 38)]:
        G = adj["Kh"]
        np.testing.assert_allclose(sym_fd("Kh", K + s * np.eye(N), i, j), G[i, j] * (1 if i == j else 2), rtol=1e-6,
                                   atol=1e-8)
    for (i, j) in [(0, 0), (2, 1), (5, 3)]:
        np.testing.assert_allclose(sym_fd("Kuu", Kuu, i, j), adj["Kuu"][i, j] * (1 if i == j else 2), rtol=1e-6,
                                   atol=1e-8)
    for (i, j) in [(0, 0), (3, 20), (5, 39)]:
        E = np.zeros_like(Kuf)
        E[i, j] = h
        np.testing.assert_allclose((f(Kuf=Kuf + E) - f(Kuf=Kuf - E)) / (2 * h), adj["Kuf"][i, j], rtol=1e-6, atol=1e-8)
    for i in (0, 11):
        E = np.zeros(N)
        E[i] = h
        np.testing.assert_allclose((f(kdiag=kd + E) - f(kdiag=kd - E)) / (2 * h), adj["kdiag"], rtol=1e-6, atol=1e-8)
    fs = lambda ss: C.bound_from(K + ss * np.eye(N), Kuf, Kuu, kd, ss, e, v)
    np.testing.assert_allclose((fs(s + h) - fs(s - h)) / (2 * h), adj["s"], rtol=1e-6)
    for (p, i) in [(0, 0), (1, 13), (1, 39)]:
        E = np.zeros_like(e)
        E[i, p] = h
        np.testing.assert_allclose((f(e=e + E) - f(e=e - E)) / (2 * h), adj["e"][i, p], rtol=1e-6, atol=1e-8)
        E = np.zeros_like(v)
        E[p, i] = h
        np.testing.assert_allclose((f(v=v + E) - f(v=v - E)) / (2 * h), adj["v"][p, i], rtol=1e-6, atol=1e-8)


# ---- the parameter-gradient oracle -------------------------------------------------------------------------------
def _kernels():
    return {
        "rbf_ard": lambda: O.SquaredExponential(variance=1.3, lengthscales=np.array([0.8, 1.4, 1.1])),
        "sum_lin_white": lambda: O.Sum([O.Matern32(variance=0.9, lengthscales=1.2), O.Linear(variance=0.3),
                                        O.White(variance=0.1)]),
        "prod_rq": lambda: O.Product([O.Matern52(variance=1.1, lengthscales=1.5),
                                      O.RationalQuadratic(variance=0.8, lengthscales=1.3, alpha=0.7)]),
        "active_dims": lambda: O.Matern52(variance=1.2, lengthscales=np.array([1.3, 0.9]), active_dims=[2, 0]),
    }


KERNELS = _kernels()
JIT = 1e-6


def _problem(name, P, N=30, M=5, D=3):
    rng = np.random.default_rng(len(name) + 10 * P)
    X = rng.standard_normal((N, D))
    Y = np.sin(X @ rng.standard_normal((D, P))) + 0.2 * rng.standard_normal((N, P))
    Z = rng.standard_normal((M, D))
    v = 0.3 * rng.standard_normal((P, N))
    mf = O.LinearMean(0.1 * rng.standard_normal((D, P)), 0.2 + 0.1 * np.arange(P))
    return X, Y, Z, v, mf, KERNELS[name]()


def _dense(X, Y, Z, v, mf, k, s):
    """The gradient from bound_adjoints on the dense K^, chained to the parameters directly."""
    N, P = Y.shape
    M = Z.shape[0]
    e = Y - mf(X)
    adj = C.bound_adjoints(k(X) + s * np.eye(N), k(Z, X), k(Z) + JIT * np.eye(M), k(X, full_cov=False), s, e, v)
    nn, _ = KG.weighted_leaf_grads(k, adj["Kh"], lambda c: c(X), lambda c: KG.leaf_dK(c, X))
    uu, uf, dg = KG.inducing_stacks(k, X, Z)
    parts = [nn, KG.reduce(adj["Kuu"], uu), KG.reduce(adj["Kuf"], uf), KG.reduce(np.full(N, adj["kdiag"]), dg)]
    leaves = [{n: sum(p[i][n] for p in parts) for n in nn[i]} for i in range(len(nn))]
    dZ = sum(np.einsum("mn,dmn->md", adj["Kuf"], st["Z"]) for st in uf)
    dZ = dZ + sum(2.0 * np.einsum("ij,dij->id", adj["Kuu"], st["Z"]) for st in uu)
    return dict(leaves=leaves, noise_variance=adj["s"], mean=KG.mean_grads(mf, X, -adj["e"]), Z=dZ, v=adj["v"])


def _flat(g):
    """Every gradient entry in a fixed order: leaf slots, noise, Z, v, mean."""
    parts = [np.ravel(np.asarray(x, dtype=np.float64)) for gd in g["leaves"] for x in gd.values()]
    parts += [np.array([g["noise_variance"]]), np.ravel(g["Z"]), np.ravel(g["v"])]
    parts += [np.ravel(g["mean"][n]) for n in sorted(g["mean"])]
    return np.concatenate(parts)


@pytest.mark.parametrize("P", [1, 2])
@pytest.mark.parametrize("name", list(KERNELS))
def test_grad_oracle_against_dense_adjoints(name, P):
    """Row blocks of 7 over N = 30 (the last one short, every diagonal block inside the loop) and the Woodbury z
    against bound_adjoints on the dense K^ and the dense solve with Q."""
    X, Y, Z, v, mf, k = _problem(name, P)
    s = 0.25
    val, g = CG.cglb_elbo_and_grad_expr(X, Y, k, Z, s, v, mean_function=mf, jitter=JIT, abs_sums=True, block_rows=7)
    ref = _dense(X, Y, Z, v, mf, k, s)
    np.testing.assert_allclose(val, C.bound(X, Y, Z, k, s, v, jitter=JIT, mean=mf(X))["elbo"], rtol=1e-12)
    a, b = _flat(g), _flat(ref)
    assert np.max(np.abs(a - b)) <= 1e-12 * np.max(np.abs(b)), np.max(np.abs(a - b)) / np.max(np.abs(b))
    # the sums of |terms| bound the gradient they scale
    for gd, ga in zip(g["leaves"], g["leaves_abs"]):
        for n in gd:
            assert np.all(np.abs(gd[n]) <= np.asarray(ga[n]) * (1 + 1e-12))
    assert abs(g["noise_variance"]) <= g["noise_abs"]
    assert np.all(np.abs(g["Z"]) <= g["Z_abs"] * (1 + 1e-12)) and np.all(np.abs(g["v"]) <= g["v_abs"] * (1 + 1e-12))
    # one block of all rows: the same numbers
    _, g1 = CG.cglb_elbo_and_grad_expr(X, Y, k, Z, s, v, mean_function=mf, jitter=JIT)
    assert np.max(np.abs(_flat(g1) - a)) <= 1e-12 * np.max(np.abs(a))


def _set(obj, name, idx, value):
    cur = getattr(obj, name)
    if np.ndim(cur) == 0:
        setattr(obj, name, value)
    else:
        arr = np.array(cur, dtype=np.float64)
        arr[idx] = value
        setattr(obj, name, arr)


@pytest.mark.parametrize("P", [1, 2])
@pytest.mark.parametrize("name", list(KERNELS))
def test_grad_oracle_against_finite_differences(name, P):
    """Central differences of cglb_oracle.bound (dense, independent of the gradient oracle) at every kernel slot, the
    noise, every entry of Z and of v, and the Linear mean's A and b."""
    X, Y, Z, v, mf, k = _problem(name, P)
    s = 0.25
    _, g = CG.cglb_elbo_and_grad_expr(X, Y, k, Z, s, v, mean_function=mf, jitter=JIT)
    state = dict(s=s, Z=Z, v=v)

    def f():
        return C.bound(X, Y, state["Z"], k, state["s"], state["v"], jitter=JIT, mean=mf(X))["elbo"]

    checks = []   # (what, get, put, analytic)
    for li, lf in enumerate(KG.leaves(k)):
        for name_, gv in g["leaves"][li].items():
            for idx in np.ndindex(np.shape(gv)):
                checks.append(((li, name_, idx), lambda lf=lf, n=name_, i=idx: float(np.asarray(getattr(lf, n))[i]),
                               lambda x, lf=lf, n=name_, i=idx: _set(lf, n, i, x), float(np.asarray(gv)[idx])))
    checks.append(("noise", lambda: state["s"], lambda x: state.__setitem__("s", x), g["noise_variance"]))
    for key in ("Z", "v"):
        for idx in np.ndindex(state[key].shape):
            def put(x, key=key, idx=idx):
                a = state[key].copy()
                a[idx] = x
                state[key] = a
            checks.append(((key, idx), lambda key=key, idx=idx: float(state[key][idx]), put, float(g[key][idx])))
    for n in ("A", "b"):
        for idx in np.ndindex(getattr(mf, n).shape):
            checks.append(((n, idx), lambda n=n, idx=idx: float(getattr(mf, n)[idx]),
                           lambda x, n=n, idx=idx: _set(mf, n, idx, x), float(g["mean"][n][idx])))
    top = max(abs(c[3]) for c in checks)
    worst = 0.0
    for what, get, put, ana in checks:
        x0 = get()
        h = 1e-5 * max(1.0, abs(x0))
        put(x0 + h)
        fu = f()
        put(x0 - h)
        fd = f()
        put(x0)
        num = (fu - fd) / (2 * h)
        err = abs(num - ana) / (1e-6 * max(abs(ana), 1e-3 * top))
        worst = max(worst, err)
        assert err <= 1.0, (what, num, ana)
    assert len(checks) > 1 + Z.size + v.size
