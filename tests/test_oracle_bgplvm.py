"""CPU pins of the Bayesian GPLVM oracles: the psi statistics against tensor-product Gauss-Hermite quadrature of the
expectations (independent of the closed forms), the gradient oracle against central finite differences of the bound,
the psi adjoints alone (psi_vjp) against central finite differences of the contracted psi statistics, pca_reduce
against the projection onto the top eigenvectors, and the argument checks of the new entry points."""
import ctypes

import numpy as np
import pytest

from gpflow_b200 import _lib
from gpflow_b200.kernels import Matern32, SquaredExponential, compile_kernel
from gpflow_b200.utilities.ops import pca_reduce
from oracle import gp_oracle as O
from tests.bgplvm_grad_oracle import bgplvm_elbo_grad, psi_vjp
from tests.bgplvm_oracle import bgplvm_elbo, psi_statistics


def _quadrature(mu, S, Z, ko, deg=60):
    """E[k(x, z)] and sum_n E[k(z, x) k(x, z')] by tensor-product Gauss-Hermite over x ~ N(mu_n, diag S_n)."""
    t, w = np.polynomial.hermite_e.hermegauss(deg)
    w = w / w.sum()
    Q = mu.shape[1]
    grids = np.meshgrid(*([t] * Q), indexing="ij")
    nodes = np.stack([g.reshape(-1) for g in grids], 1)
    weights = np.prod(np.meshgrid(*([w] * Q), indexing="ij"), axis=0).reshape(-1)
    psi1 = np.empty((mu.shape[0], Z.shape[0]))
    psi2 = np.zeros((Z.shape[0],) * 2)
    for n in range(mu.shape[0]):
        X = mu[n] + np.sqrt(S[n]) * nodes
        K = ko(X, Z)
        psi1[n] = weights @ K
        psi2 += (K * weights[:, None]).T @ K
    return psi1, psi2


@pytest.mark.parametrize("Q, ls, ad", [(1, 0.8, None), (2, 1.1, None), (2, np.array([0.7, 1.6]), None),
                                       (3, np.array([0.9, 1.3]), [2, 0])])
def test_psi_statistics_match_quadrature(Q, ls, ad):
    rng = np.random.default_rng(Q)
    N, M = 4, 5
    mu, S, Z = rng.standard_normal((N, Q)), rng.uniform(0.05, 0.6, (N, Q)), rng.standard_normal((M, Q))
    ko = O.SquaredExponential(1.4, ls, active_dims=ad)
    cols = np.arange(Q) if ad is None else np.asarray(ad)
    q1, q2 = _quadrature(mu[:, cols], S[:, cols], Z[:, cols], O.SquaredExponential(1.4, ls))
    p0, p1, p2 = psi_statistics(mu, S, Z, ko)
    assert p0 == pytest.approx(N * 1.4)
    np.testing.assert_allclose(p1, q1, rtol=0, atol=1e-12)
    np.testing.assert_allclose(p2, q2, rtol=0, atol=1e-12)


def _fd_case(ls, ad, Q=3, seed=0):
    rng = np.random.default_rng(seed)
    N, M, P = 8, 5, 2
    d = dict(Y=rng.standard_normal((N, P)), mu=rng.standard_normal((N, Q)), S=rng.uniform(0.1, 0.9, (N, Q)),
             Z=rng.standard_normal((M, Q)), m0=0.1 * rng.standard_normal((N, Q)), p0=rng.uniform(0.5, 2.0, (N, Q)))
    return d, O.SquaredExponential(1.3, ls, active_dims=ad)


@pytest.mark.parametrize("ls, ad", [(0.9, None), (np.array([0.8, 1.4, 1.1]), None), (np.array([0.8, 1.4]), [2, 0])])
def test_gradient_oracle_matches_finite_differences(ls, ad):
    d, ko = _fd_case(ls, ad)
    g = bgplvm_elbo_grad(d["Y"], d["mu"], d["S"], d["Z"], ko, 0.3, d["m0"], d["p0"])
    h = 1e-6

    def f(noise=0.3, k=ko, **kw):
        a = {**d, **kw}
        return bgplvm_elbo(a["Y"], a["mu"], a["S"], a["Z"], k, noise, a["m0"], a["p0"])

    def close(got, fd):
        np.testing.assert_allclose(got, fd, rtol=1e-6, atol=1e-6 * max(1.0, np.max(np.abs(fd))))

    close(g["noise"], (f(0.3 + h) - f(0.3 - h)) / (2 * h))
    mk = lambda v, l: O.SquaredExponential(v, l, active_dims=ad)
    close(g["variance"], (f(k=mk(1.3 + h, ls)) - f(k=mk(1.3 - h, ls))) / (2 * h))
    ll = np.atleast_1d(np.asarray(ls, dtype=float))
    fd = []
    for i in range(ll.size):
        e = np.zeros_like(ll)
        e[i] = h
        fd.append((f(k=mk(1.3, (ll + e) if np.ndim(ls) else float(ll[0] + h)))
                   - f(k=mk(1.3, (ll - e) if np.ndim(ls) else float(ll[0] - h)))) / (2 * h))
    close(np.atleast_1d(g["lengthscales"]), np.array(fd))
    for name in ("mu", "S", "Z"):
        arr = d[name]
        fd = np.zeros_like(arr)
        for idx in np.ndindex(arr.shape):
            ap, am = arr.copy(), arr.copy()
            ap[idx] += h
            am[idx] -= h
            fd[idx] = (f(**{name: ap}) - f(**{name: am})) / (2 * h)
        close(g[name], fd)


@pytest.mark.parametrize("kind", ["scalar", "ard", "active_dims"])
@pytest.mark.parametrize("nd", [1, 3, 9])
def test_psi_vjp_matches_finite_differences(nd, kind):
    """psi_vjp against central differences of F = sum G1 * psi1 + sum G2 * psi2 (psi_statistics, the Cholesky forms)
    at every element of mu, S, Z and at the variance and each lengthscale, with G1 and G2 of mixed signs."""
    rng = np.random.default_rng(100 * nd + len(kind))
    N, M = 5, 4
    Q = nd + 2 if kind == "active_dims" else nd
    ad = list(rng.permutation(Q)[:nd]) if kind == "active_dims" else None
    ls = 0.9 if kind == "scalar" else rng.uniform(0.6, 1.8, nd)
    mu, S, Z = rng.standard_normal((N, Q)), rng.uniform(0.05, 0.8, (N, Q)), rng.standard_normal((M, Q))
    G1 = rng.standard_normal((N, M))
    G2 = rng.standard_normal((M, M))
    G2 = G2 + G2.T
    ko = O.SquaredExponential(1.3, ls, active_dims=ad)
    g = psi_vjp(mu, S, Z, ko, G1, G2)
    # the block-wise evaluation does not depend on the block size
    g1 = psi_vjp(mu, S, Z, ko, G1, G2, block_elems=1)
    for k in g:
        np.testing.assert_allclose(g1[k], g[k], rtol=1e-13, atol=1e-15)
    h = 1e-6

    def f(mu=mu, S=S, Z=Z, k=ko):
        _, p1, p2 = psi_statistics(mu, S, Z, k)
        return float(np.sum(G1 * p1) + np.sum(G2 * p2))

    def close(got, fd):
        np.testing.assert_allclose(got, fd, rtol=1e-6, atol=1e-7 * max(1.0, np.max(np.abs(fd))))

    for name, arr in (("mu", mu), ("S", S), ("Z", Z)):
        fd = np.zeros_like(arr)
        for idx in np.ndindex(arr.shape):
            ap, am = arr.copy(), arr.copy()
            ap[idx] += h
            am[idx] -= h
            fd[idx] = (f(**{name: ap}) - f(**{name: am})) / (2 * h)
        close(g[name], fd)
    mk = lambda v, l: O.SquaredExponential(v, l, active_dims=ad)
    close(g["variance"], (f(k=mk(1.3 + h, ls)) - f(k=mk(1.3 - h, ls))) / (2 * h))
    if kind == "scalar":  # one lengthscale shared by the active dims: its derivative is the sum over the dims
        close(np.sum(g["lengthscales"]), (f(k=mk(1.3, ls + h)) - f(k=mk(1.3, ls - h))) / (2 * h))
    else:
        fd = [(f(k=mk(1.3, ls + h * e)) - f(k=mk(1.3, ls - h * e))) / (2 * h) for e in np.eye(nd)]
        close(g["lengthscales"], np.array(fd))


def test_psi_vjp_abs_sums_bound_the_values():
    """The magnitude sums of psi_vjp: T >= |value| everywhere, zero outside the active dims, U the largest exponent."""
    rng = np.random.default_rng(4)
    N, Q, M = 6, 4, 3
    mu, S, Z = rng.standard_normal((N, Q)), rng.uniform(0.05, 0.8, (N, Q)), rng.standard_normal((M, Q))
    mu[0] += 20.0  # one point far from every inducing point: psi2 exponents of a few hundred
    G2 = rng.standard_normal((M, M))
    ko = O.SquaredExponential(1.1, np.array([0.8, 1.2]), active_dims=[3, 1])
    g, sums = psi_vjp(mu, S, Z, ko, rng.standard_normal((N, M)), G2 + G2.T, abs_sums=True)
    for k, (T, U, C) in sums.items():
        assert np.all(T >= np.abs(g[k]) * (1 - 1e-12)) and np.all(C >= 0), k
        assert np.all(np.asarray(U) >= 0) and np.all(np.asarray(U) < 3000), k
    for k in ("mu", "S", "Z"):
        assert not np.any(sums[k][0][:, [0, 2]]) and not np.any(g[k][:, [0, 2]])
    # the largest exponent behind dmu of the far point is its largest psi2 exponent (about twice its psi1 exponents)
    c, l2 = [3, 1], np.array([0.8, 1.2]) ** 2
    zb, ez = 0.5 * (Z[:, None, c] + Z[None, :, c]), np.sum((Z[:, None, c] - Z[None, :, c]) ** 2 / (4 * l2), -1)
    u2 = ez + 0.5 * np.sum(np.log1p(2 * S[0, c] / l2)) + np.sum((mu[0, c] - zb) ** 2 / (l2 + 2 * S[0, c]), -1)
    assert sums["mu"][1][0, 1] == pytest.approx(u2.max(), rel=1e-12) and u2.max() > 300 > sums["mu"][1][1:, 1].max()


def test_pca_reduce_projects_onto_top_eigenvectors():
    rng = np.random.RandomState(999)
    Y = rng.randn(30, 5) @ rng.randn(5, 5)
    X = pca_reduce(Y, 2)
    Yc = Y - Y.mean(0)
    evals, evecs = np.linalg.eig(np.cov(Y, rowvar=False))
    top = evecs[:, np.argsort(evals)[::-1][:2]][:, ::-1]  # ascending order of the two largest, as eigh returns them
    ref = Yc @ top
    for q in range(2):
        assert np.allclose(X[:, q], ref[:, q]) or np.allclose(X[:, q], -ref[:, q])
    with pytest.raises(ValueError):
        pca_reduce(Y, 6)


def _call_psi(kernel, Q=2, N=4, M=3):
    lib = _lib.load()
    p = ctypes.c_void_p(16)
    return lib.gpk_rbf_psi(*compile_kernel(kernel, Q), p, p, N, Q, p, M, Q, p, p, p, p, None)


def _call_psi_grad(kernel, Q=2, N=4, M=3, ldz=None, ldg1=None, ldg2=None, null=None):
    """gpk_debug_rbf_psi_grad with placeholder pointers (the refusals return before any device work); null: the index
    of the pointer argument among (mu, S, Z, G1t, G2, dmu, dS, dZ, gpar, ws) passed as NULL."""
    lib = _lib.load()
    ptrs = [ctypes.c_void_p(16) if i != null else None for i in range(10)]
    mu, S, Z, G1t, G2, dmu, dS, dZ, gpar, ws = ptrs
    geom = (ctypes.c_int64 * 9)()
    return lib.gpk_debug_rbf_psi_grad(*compile_kernel(kernel, Q), mu, S, N, Q, Z, M, Q if ldz is None else ldz, G1t,
                                      N if ldg1 is None else ldg1, G2, M if ldg2 is None else ldg2, dmu, dS, dZ, gpar,
                                      ws, geom, None)


def test_entry_points_reject_bad_arguments():
    lib = _lib.load()
    assert _call_psi(Matern32()) == -1 and b"one SquaredExponential leaf" in lib.gpk_last_error()
    assert _call_psi(SquaredExponential() + SquaredExponential()) == -1
    assert _call_psi(SquaredExponential(), Q=33) == -1 and b"at most 32" in lib.gpk_last_error()
    assert _call_psi(SquaredExponential(), N=0) == -1 and b"bad sizes" in lib.gpk_last_error()
    p = ctypes.c_void_p(16)
    k = compile_kernel(SquaredExponential(), 2)
    out = lib.gpk_bgplvm_elbo(*k, p, p, 4, 2, p, 1, p, 3, 2, p, p, 0.0, 1e-6, p, p, None)
    assert out == -1 and b"noise variance must be positive" in lib.gpk_last_error()
    out = lib.gpk_bgplvm_elbo_grad(*k, p, p, 4, 2, p, 1, p, 3, 2, p, p, 0.5, 1e-6, p, 64, None, p, p, p, None)
    assert out == -1 and b"dmu, dS and dZ are required" in lib.gpk_last_error()
    out = lib.gpk_bgplvm_elbo_grad(*k, p, p, 4, 2, p, 1, p, 3, 2, p, p, 0.5, 1e-6, p, 5, p, p, p, p, None)
    assert out == -1 and b"n_out" in lib.gpk_last_error()
    assert lib.gpk_bgplvm_elbo_grad_ws(100, 3, 10, 2) > lib.gpk_bgplvm_elbo_ws(100, 3, 10, 2) > lib.gpk_rbf_psi_ws(100, 10)
    # the psi adjoints alone: the refusals of gpk_rbf_psi, and leading dimensions of G1t and G2 below N and M
    assert _call_psi_grad(Matern32()) == -1 and b"one SquaredExponential leaf" in lib.gpk_last_error()
    assert _call_psi_grad(SquaredExponential() + SquaredExponential()) == -1
    assert _call_psi_grad(SquaredExponential(), Q=33) == -1 and b"at most 32" in lib.gpk_last_error()
    assert _call_psi_grad(SquaredExponential(), M=65536) == -1 and b"at most 65535" in lib.gpk_last_error()
    assert _call_psi_grad(SquaredExponential(), N=0) == -1 and b"bad sizes" in lib.gpk_last_error()
    assert _call_psi_grad(SquaredExponential(), ldz=1) == -1 and b"bad sizes" in lib.gpk_last_error()
    assert _call_psi_grad(SquaredExponential(), ldg1=3) == -1 and b"bad sizes" in lib.gpk_last_error()
    assert _call_psi_grad(SquaredExponential(), ldg2=2) == -1 and b"bad sizes" in lib.gpk_last_error()
    assert _call_psi_grad(SquaredExponential(), null=9) == -1 and b"NULL" in lib.gpk_last_error()
