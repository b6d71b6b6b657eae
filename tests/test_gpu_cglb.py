"""CGLB on the device: the matrix-free product gpk_kmv against the oracle within a bar derived from the K-build's element
intervals (tests/kbuild_bounds.py) plus the summation depth, its determinism and an N = 2^17 case against row blocks of
the K-build; the device CG loop against tests/cglb_oracle.py (iteration count, v, restarts, warm start); the bound at
the device's v; the reference's tests (tests/gpflow/models/test_cglb.py) on the device model; memory at N = 2^17; and
the refusals; and the gradient element by element against tests/cglb_grad_oracle.py at several outputs, in CG mode and at
N > 2^14.  Every direct device call has a sentinel guard region behind its output and workspace."""
import time

import numpy as np
import pytest

import gpflow_b200 as gpf
from gpflow_b200 import _lib, ops
from oracle import gp_oracle as O
from tests import cglb_grad_oracle as CGO
from tests import cglb_oracle as C
from tests import helpers as H
from tests import kbuild_bounds as B

pytestmark = pytest.mark.gpu
U = 2.0 ** -53
SENT = -7.25e300
GUARD = 512


def _T():
    import torch
    return torch


def _guarded(n):
    """A device fp64 buffer of n elements followed by GUARD sentinels; returns (view, full)."""
    T = _T()
    full = T.full((n + GUARD,), SENT, dtype=T.float64, device="cuda")
    return full[:n], full


def _guard_ok(full, n):
    assert bool((full[n:] == SENT).all()), "a device call wrote past its buffer"


def _kmv(desc, X, X2, V, diag=0.0, ldv=None, ldo=None):
    """gpk_kmv on host arrays with guarded output / workspace; returns out [N, P] (NumPy)."""
    lib = _lib.load()
    T = _T()
    N, D = X.shape
    P = V.shape[1]
    N2 = N if X2 is None else X2.shape[0]
    ldv = ldv or P
    ldo = ldo or P
    Vp = np.zeros((N2, ldv))
    Vp[:, :P] = V
    Xd = T.from_numpy(np.ascontiguousarray(X)).cuda()
    X2d = None if X2 is None else T.from_numpy(np.ascontiguousarray(X2)).cuda()
    Vd = T.from_numpy(Vp).cuda()
    out, ofull = _guarded(N * ldo)
    wsn = (lib.gpk_kmv_ws(N, N2, P) + 7) // 8
    ws, wfull = _guarded(wsn)
    _lib.check(lib.gpk_kmv(*desc, ops._p(Xd), N, D, None if X2d is None else ops._p(X2d), N2, D, D, ops._p(Vd), P, ldv,
                           diag, ops._p(out), ldo, ops._p(ws), ops._stream()), "gpk_kmv")
    T.cuda.synchronize()
    _guard_ok(ofull, N * ldo)
    _guard_ok(wfull, wsn)
    return out.cpu().numpy().reshape(N, ldo)[:, :P].copy()


EXPRS = ["rbf", "rbf_ard", "m12", "m32", "m52", "exp", "lin", ("sum", "rbf", "lin"),
         ("prod", "m32", ("rbf_ard", [0, 2])), ("sum", ("m52", [1]), ("prod", "m32", "exp"))]


def _kmv_bar(desc, X, X2, V, diag):
    cen, lo, hi = B.expr_interval(desc, X, X2, dtype=np.float64)
    w = np.maximum(hi - cen, cen - lo)
    if X2 is None:
        cen = cen + diag * np.eye(X.shape[0])
    N2 = cen.shape[1]
    gam = (N2 // 16 + 80) * U * 1.01
    return cen @ V, w @ np.abs(V) + gam * (np.abs(cen) @ np.abs(V)) + U * np.abs(cen @ V)


@pytest.mark.parametrize("expr", EXPRS, ids=str)
@pytest.mark.parametrize("shape", [(200, None, 1), (333, 517, 3), (1000, None, 8), (77, 1500, 9), (5000, None, 1)])
def test_kmv_against_oracle(expr, shape):
    N, N2, P = shape
    D = 3
    rng = np.random.default_rng(N + P)
    X = rng.standard_normal((N, D))
    X2 = None if N2 is None else rng.standard_normal((N2, D))
    V = rng.standard_normal((N if N2 is None else N2, P))
    kg, = H.build(expr, D, [gpf.kernels])
    desc = gpf.kernels.compile_kernel(kg, D)
    diag = 0.37 if N2 is None else 0.0
    dev = _kmv(desc, X, X2, V, diag, ldv=P + (1 if P == 3 else 0), ldo=P + (2 if P == 9 else 0))
    ref, bar = _kmv_bar(desc, X, X2, V, diag)
    ratio = np.max(np.abs(dev - ref) / bar)
    print(f"kmv {expr} {shape}: max error / bar = {ratio:.3g}")
    assert ratio <= 1.0
    assert np.array_equal(dev, _kmv(desc, X, X2, V, diag, ldv=P + (1 if P == 3 else 0), ldo=P + (2 if P == 9 else 0)))


def test_kmv_large_against_kbuild_rows():
    """N = 2^17, D = 8, P = 1: three row blocks of K(X, X) from gpk_kbuild (the fast path) times V."""
    T = _T()
    N, D, P = 1 << 17, 8, 1
    rng = np.random.default_rng(7)
    X = rng.standard_normal((N, D)) * 0.7
    V = rng.standard_normal((N, P))
    kg = gpf.kernels.SquaredExponential(variance=1.3, lengthscales=1.9)
    desc = gpf.kernels.compile_kernel(kg, D)
    dev = _kmv(desc, X, None, V, 0.1)
    assert np.array_equal(dev, _kmv(desc, X, None, V, 0.1))
    Xd = T.from_numpy(X).cuda()
    Vd = T.from_numpy(V).cuda()
    worst = 0.0
    for r0 in (0, 61440, N - 4096):
        Kb = kg.K(Xd[r0:r0 + 4096], Xd)
        ref = (Kb @ Vd).cpu().numpy() + 0.1 * V[r0:r0 + 4096]
        bar = ((N // 16 + 80) * U + 64 * U) * (Kb.abs() @ Vd.abs()).cpu().numpy() + 2 * U * np.abs(ref)
        worst = max(worst, float(np.max(np.abs(dev[r0:r0 + 4096] - ref) / bar)))
    print(f"kmv N=2^17 against kbuild rows: max error / bar = {worst:.3g}")
    assert worst <= 1.0


# ---- the model ---------------------------------------------------------------------------------------------------
def _reg(N, M, D=2, seed=0):
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((N, D))
    Y = np.sin(X @ np.linspace(-1.4, 0.5, D)[:, None]) + 0.3 * rng.standard_normal((N, 1))
    return X, Y, rng.standard_normal((M, D))


def _pair(expr, D):
    kg, ko = H.build(expr, D, [gpf.kernels, O])
    return kg, ko


def _margin(rz, tol):
    """The oracle's final 0.5 rz must clear the threshold by >= 1e-6 relative for the counts to be comparable."""
    assert abs(0.5 * rz - tol) >= 1e-6 * tol, (rz, tol)


@pytest.mark.parametrize("restart", [40, 3])
@pytest.mark.parametrize("expr", ["rbf", "m52", ("sum", "rbf", "lin")], ids=str)
def test_cg_against_oracle(expr, restart):
    # a well-conditioned system (s = 0.5, 40 inducing points): the recursive residual stays close to e - K^ v, so
    # the warm start below meets the tolerance at once, as it does in the oracle
    X, Y, Z = _reg(700, 40, D=2, seed=3)
    kg, ko = _pair(expr, 2)
    s = 0.5
    tol = 1e-4
    v_ref, it_ref, rz_ref = C.run_cg(X, Y, Z, ko, s, np.zeros((1, 700)), tol, 100, restart)
    _margin(rz_ref, tol)
    m = gpf.models.CGLB((X, Y), kernel=kg, inducing_variable=Z, noise_variance=s, cg_tolerance=tol,
                        restart_cg_iters=restart)
    e1 = float(m.elbo())
    assert m.cg_iterations() == it_ref
    v = m.aux_vec.numpy()
    assert np.linalg.norm(v - v_ref) <= 1e-9 * np.linalg.norm(v_ref)
    ref = C.bound(X, Y, Z, ko, s, v)
    np.testing.assert_allclose(e1, ref["elbo"], rtol=1e-11)
    for i, k in ((1, "const"), (2, "logdet"), (3, "quad")):
        np.testing.assert_allclose(float(m.elbo_terms()[i - 1]), ref[k], rtol=1e-11)
    # warm start at the converged v: no step, the same bits
    e2 = m.elbo()
    assert m.cg_iterations() == 0 and float(e2) == e1


@pytest.mark.parametrize("M", [17, 64, 200])
@pytest.mark.parametrize("expr", ["rbf", "m12", "rq", ("prod", "m32", "rbf_ard")], ids=str)
def test_bound_at_given_v(expr, M):
    """Trainable v (no CG), any P: the bound against the oracle at a random v."""
    rng = np.random.default_rng(M)
    N, D, P = 900, 3, 2
    X = rng.standard_normal((N, D))
    Y = rng.standard_normal((N, P))
    Z = rng.standard_normal((M, D))
    kg, ko = _pair(expr, D)
    m = gpf.models.CGLB((X, Y), kernel=kg, inducing_variable=Z, noise_variance=0.3, v_grad_optimization=True)
    v = 0.1 * rng.standard_normal((P, N))
    m.aux_vec.assign(v)
    ref = C.bound(X, Y, Z, ko, 0.3, v)
    np.testing.assert_allclose(float(m.elbo()), ref["elbo"], rtol=2e-10)
    np.testing.assert_allclose(float(m._last[5]), ref["rz"], rtol=1e-9)


def _ref_data():
    rng = np.random.RandomState(999)
    n, t, d = 100, 20, 2
    x = rng.randn(n, d)
    xs = rng.randn(t, d)
    y = np.sin(x @ np.array([[-1.4], [0.5]]) + 0.5 * rng.randn(n, 1))
    return (x, y), rng.randn(10, 2), xs


def test_reference_basics_and_guarantees():
    (x, y), z, _ = _ref_data()
    se = gpf.kernels.SquaredExponential
    sgpr = gpf.models.SGPR((x, y), kernel=se(), inducing_variable=z, noise_variance=0.2)
    cglb = gpf.models.CGLB((x, y), kernel=se(), inducing_variable=z, noise_variance=0.2, v_grad_optimization=True)
    cglb.elbo()
    sgpr.elbo()
    np.testing.assert_allclose(float(cglb.elbo_terms()[2]), float(sgpr.elbo_terms()[2]), rtol=1e-12)
    assert float(cglb.elbo_terms()[1]) >= float(sgpr.elbo_terms()[1])
    K = O.SquaredExponential().K(x) + 0.2 * np.eye(100)
    assert float(cglb.elbo_terms()[1]) <= -0.5 * np.linalg.slogdet(K)[1]
    # the CG quad term: below the Cholesky one and within the tolerance of it
    K = O.SquaredExponential().K(x) + 1e-2 * np.eye(100)
    chol_quad = -0.5 * (y.T @ np.linalg.solve(K, y)).item()
    m = gpf.models.CGLB((x, y), kernel=se(), inducing_variable=z, noise_variance=1e-2, cg_tolerance=1e-2,
                        max_cg_iters=100, restart_cg_iters=10)
    m.elbo()
    q = float(m.elbo_terms()[2])
    assert q <= chol_quad and abs(q - chol_quad) <= 1e-2
    gpr = gpf.models.GPR((x, y), kernel=se(), noise_variance=1e-2)
    assert float(m.elbo()) <= float(gpr.log_marginal_likelihood())


def test_reference_predict():
    (x, y), z, xs = _ref_data()
    se = gpf.kernels.SquaredExponential
    gpr = gpf.models.GPR((x, y), kernel=se(), noise_variance=0.2)
    sgpr = gpf.models.SGPR((x, y), kernel=se(), inducing_variable=z, noise_variance=0.2)
    cglb = gpf.models.CGLB((x, y), kernel=se(), inducing_variable=z, noise_variance=0.2)
    gm, _ = gpr.predict_y(xs)
    sm, sv = sgpr.predict_y(xs)
    cm, cv = cglb.predict_y(xs, cg_tolerance=1e6)
    np.testing.assert_allclose(H.to_np(cm), H.to_np(sm), rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(H.to_np(cv), H.to_np(sv), rtol=1e-10, atol=1e-12)
    cm, _ = cglb.predict_y(xs, cg_tolerance=1e-12)
    assert np.allclose(H.to_np(gm), H.to_np(cm))
    assert not np.any(cglb.aux_vec.numpy())  # prediction does not store its CG result
    v, _, _ = C.run_cg(x, y, z, O.SquaredExponential(), 0.2, np.zeros((1, 100)), 1e-3, 100, 40)
    om, ov = C.predict_f(x, y, z, O.SquaredExponential(), 0.2, v, xs)
    fm, fv = cglb.predict_f(xs)
    np.testing.assert_allclose(H.to_np(fm), om, rtol=1e-8, atol=1e-10)
    np.testing.assert_allclose(H.to_np(fv), ov, rtol=1e-10, atol=1e-12)


def test_cg_raises_the_bound_below_gpr():
    X, Y, Z = _reg(400, 12, seed=5)
    se = gpf.kernels.SquaredExponential
    m = gpf.models.CGLB((X, Y), kernel=se(), inducing_variable=Z, noise_variance=0.1, cg_tolerance=1e-2)
    e0 = float(gpf.models.SGPR((X, Y), kernel=se(), inducing_variable=Z, noise_variance=0.1).elbo())
    e1 = float(m.elbo())
    gpr = float(gpf.models.GPR((X, Y), kernel=se(), noise_variance=0.1).log_marginal_likelihood())
    assert e0 <= e1 + 1e-9 and e1 <= gpr


def test_memory_at_2_17():
    T = _T()
    N, M, D = 1 << 17, 1024, 8
    rng = np.random.default_rng(11)
    X = rng.standard_normal((N, D))
    Y = np.sin(X[:, :1]) + 0.1 * rng.standard_normal((N, 1))
    Z = X[rng.choice(N, M, replace=False)]
    m = gpf.models.CGLB((X, Y), kernel=gpf.kernels.SquaredExponential(lengthscales=2.0), inducing_variable=Z,
                        noise_variance=0.1, max_cg_iters=2)
    T.cuda.synchronize()
    T.cuda.reset_peak_memory_stats()
    base = T.cuda.memory_allocated()
    e = float(m.elbo())
    peak = T.cuda.max_memory_allocated() - base
    lib = _lib.load()
    ws = lib.gpk_cglb_elbo_ws(N, M, 1)
    formula = 8 * (N * (M + 8 * 1) + 6 * M * M) + 8 * N * 4 + (64 << 20)
    print(f"N=2^17 M=1024: elbo {e:.6g}, workspace {ws / 2**30:.3f} GiB, peak {peak / 2**30:.3f} GiB")
    assert np.isfinite(e) and m.cg_iterations() == 2
    assert ws <= formula
    assert peak < 16 * 2 ** 30


def test_refusals():
    X, Y, Z = _reg(50, 5)
    se = gpf.kernels.SquaredExponential
    Y2 = np.hstack([Y, Y])
    m = gpf.models.CGLB((X, Y2), kernel=se(), inducing_variable=Z)
    with pytest.raises(ValueError, match="one output"):
        m.elbo()
    with pytest.raises(ValueError, match="one output"):
        m.predict_f(X[:3])
    m.predict_f(X[:3], cg_tolerance=None)  # the stored v takes any P
    m2 = gpf.models.CGLB((X, Y2), kernel=se(), inducing_variable=Z, v_grad_optimization=True)
    assert np.isfinite(float(m2.elbo()))
    m1 = gpf.models.CGLB((X, Y), kernel=se(), inducing_variable=Z)
    with pytest.raises(NotImplementedError):
        m1.predict_f(X[:3], full_output_cov=True)
    m32 = gpf.models.CGLB((X, Y), kernel=se(), inducing_variable=Z)
    m32.data = (ops.to_device(X, dtype=np.float32), ops.to_device(Y, dtype=np.float32))
    with pytest.raises(NotImplementedError, match="float64"):
        m32.elbo()
    mp = gpf.models.CGLB((X, Y), kernel=se(), inducing_variable=Z)
    mp.kernel.variance.prior = "a prior"
    with pytest.raises(NotImplementedError, match="prior"):
        mp.elbo()


# ---- the gradient ------------------------------------------------------------------------------------------------
def _entries(p):
    a = np.asarray(p.numpy())
    if a.ndim == 0:
        return [()]
    flat = [np.unravel_index(i, a.shape) for i in (0, a.size // 3, a.size - 1)]
    return list(dict.fromkeys(flat))


def _fd_check(m, grads, h=1e-6, rtol=2e-5):
    """Central differences of the device bound (trainable v: a smooth function) in every trainable parameter."""
    worst = 0.0
    for p in m.trainable_parameters:
        g = np.asarray(grads[p] if not hasattr(grads[p], "cpu") else grads[p].cpu().numpy())
        base = np.array(p.numpy(), dtype=np.float64)
        scale = max(np.max(np.abs(g)), 1.0)
        for idx in _entries(p):
            step = h * max(1.0, abs(float(base[idx])))
            up, dn = base.copy(), base.copy()
            up[idx] += step
            dn[idx] -= step
            p.assign(up)
            fu = float(m.elbo())
            p.assign(dn)
            fd = float(m.elbo())
            p.assign(base)
            num = (fu - fd) / (2 * step)
            err = abs(num - float(g[idx])) / (rtol * scale)
            worst = max(worst, err)
            assert err <= 1.0, (p.name, idx, num, float(g[idx]))
    return worst


@pytest.mark.parametrize("M", [17, 64, 200])
@pytest.mark.parametrize("expr", ["rbf", "m32", ("sum", "rbf_ard", "lin"), ("prod", "m52", "rq")], ids=str)
def test_gradient_against_finite_differences(expr, M):
    """Trainable v: every gradient (kernel slots, noise, Z, the Linear mean function, v) against central differences
    of the device bound."""
    rng = np.random.default_rng(M + 1)
    N, D = 400, 3
    X = rng.standard_normal((N, D))
    Y = np.sin(X[:, :1]) + 0.2 * rng.standard_normal((N, 1))
    Z = rng.standard_normal((M, D))
    kg, _ = _pair(expr, D)
    mf = gpf.mean_functions.Linear(A=0.1 * np.ones((D, 1)), b=np.array([0.2]))
    m = gpf.models.CGLB((X, Y), kernel=kg, inducing_variable=Z, noise_variance=0.3, mean_function=mf,
                        v_grad_optimization=True)
    m.aux_vec.assign(0.05 * rng.standard_normal((1, N)))
    _, grads = m.elbo_and_grad()
    print(f"grad FD {expr} M={M}: worst error / bar = {_fd_check(m, grads):.3g}")


def test_gradient_in_cg_mode_equals_fixed_v():
    """With CG the gradient is the trainable-v gradient at the v CG chose (v held fixed), bit for bit in the value."""
    X, Y, Z = _reg(500, 30, seed=9)
    se = gpf.kernels.Matern52
    a = gpf.models.CGLB((X, Y), kernel=se(), inducing_variable=Z, noise_variance=0.2, cg_tolerance=1e-3)
    ea, ga = a.elbo_and_grad()
    assert a.cg_iterations() > 0
    b = gpf.models.CGLB((X, Y), kernel=se(), inducing_variable=Z, noise_variance=0.2, v_grad_optimization=True)
    b.aux_vec.assign(a.aux_vec.numpy())
    eb, gb = b.elbo_and_grad()
    np.testing.assert_allclose(float(ea), float(eb), rtol=1e-12)
    for pa, pb in zip(a.trainable_parameters, [p for p in b.trainable_parameters if p is not b.aux_vec]):
        np.testing.assert_allclose(np.asarray(ga[pa]), np.asarray(gb[pb]), rtol=1e-9, atol=1e-9)
    assert a.aux_vec not in ga


def test_scipy_cg_mode_raises_the_bound():
    X, Y, Z = _reg(300, 15, seed=2)
    m = gpf.models.CGLB((X, Y), kernel=gpf.kernels.SquaredExponential(), inducing_variable=Z, noise_variance=0.5,
                        cg_tolerance=1e-3)
    e0 = float(m.elbo())
    gpf.optimizers.Scipy().minimize(m.training_loss_closure(), m.trainable_variables, options=dict(maxiter=30))
    e1 = float(m.elbo())
    gpr = gpf.models.GPR((X, Y), kernel=m.kernel, noise_variance=float(m.likelihood.variance.numpy()))
    assert e1 > e0 and e1 <= float(gpr.log_marginal_likelihood())


def test_scipy_trainable_v_against_oracle_lbfgs():
    """L-BFGS-B with trainable v from the device gradient against the same optimiser on the oracle's bound and its
    closed-form gradient (noise, kernel variance and lengthscale, v; Z fixed)."""
    from scipy.optimize import minimize
    X, Y, Z = _reg(120, 8, seed=6)
    N = X.shape[0]
    m = gpf.models.CGLB((X, Y), kernel=gpf.kernels.SquaredExponential(), inducing_variable=Z, noise_variance=0.5,
                        v_grad_optimization=True)
    gpf.utilities.set_trainable(m.inducing_variable, False)
    gpf.optimizers.Scipy().minimize(m.training_loss_closure(), m.trainable_variables, options=dict(maxiter=60))
    dev = float(m.elbo())

    def neg(u):
        var, ls, s = np.exp(u[:3])
        v = u[3:][None, :]
        ko = O.SquaredExponential(var, ls)
        return -C.bound(X, Y, Z, ko, s, v)["elbo"]

    u0 = np.concatenate([np.log([1.0, 1.0, 0.5]), np.zeros(N)])
    res = minimize(neg, u0, method="L-BFGS-B", options=dict(maxiter=60))
    assert dev >= -res.fun - 1e-3 * abs(res.fun)


def test_adam_trainable_v_no_host_to_device_copy():
    import torch
    from torch.profiler import ProfilerActivity, profile
    X, Y, Z = _reg(400, 20, seed=4)
    m = gpf.models.CGLB((X, Y), kernel=gpf.kernels.SquaredExponential(), inducing_variable=Z, noise_variance=0.5,
                        v_grad_optimization=True)
    opt = gpf.optimizers.Adam(0.01)
    e0 = float(m.elbo())
    opt.minimize(m.training_loss, m.trainable_variables)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            opt.minimize(m.training_loss, m.trainable_variables)
        torch.cuda.synchronize()
    h2d = [e.key for e in prof.key_averages() if "HtoD" in e.key or "Memcpy HtoD" in e.key]
    assert not h2d, h2d
    assert float(m.elbo()) > e0


def test_elbo_and_grad_memory_at_2_17():
    T = _T()
    N, M, D = 1 << 17, 1024, 8
    rng = np.random.default_rng(12)
    X = rng.standard_normal((N, D))
    Y = np.sin(X[:, :1]) + 0.1 * rng.standard_normal((N, 1))
    Z = X[rng.choice(N, M, replace=False)]
    m = gpf.models.CGLB((X, Y), kernel=gpf.kernels.SquaredExponential(lengthscales=2.0), inducing_variable=Z,
                        noise_variance=0.1, max_cg_iters=2)
    T.cuda.synchronize()
    T.cuda.reset_peak_memory_stats()
    base = T.cuda.memory_allocated()
    e, g = m.elbo_and_grad(device_arrays=True)
    peak = T.cuda.max_memory_allocated() - base
    ws = _lib.load().gpk_cglb_elbo_grad_ws(N, M, 1)
    formula = 8 * (N * (3 * M + 12 * 1 + 4) + 10 * M * M) + (64 << 20)
    print(f"elbo_and_grad N=2^17 M=1024: workspace {ws / 2**30:.3f} GiB, peak {peak / 2**30:.3f} GiB")
    assert np.isfinite(float(e)) and np.all(np.isfinite(g[m.inducing_variable.Z].cpu().numpy()))
    assert ws <= formula and peak < 16 * 2 ** 30


@pytest.mark.parametrize("run_cg", [0, 1])
def test_cglb_entry_points_guarded(run_cg):
    """gpk_cglb_elbo and gpk_cglb_elbo_grad called directly with a guard region behind out, v, dZ, dv and the workspace."""
    T = _T()
    lib = _lib.load()
    X, Y, Z = _reg(333, 21, seed=1)
    N, D = X.shape
    M = Z.shape[0]
    kg = gpf.kernels.Matern32()
    desc = gpf.kernels.compile_kernel(kg, D)
    Xd, Yd, Zd = (T.from_numpy(a).cuda() for a in (X, Y, Z))
    ref = None
    for grad in (False, True):
        v, vf = _guarded(N)
        v.zero_()
        nws = ((lib.gpk_cglb_elbo_grad_ws if grad else lib.gpk_cglb_elbo_ws)(N, M, 1) + 7) // 8
        ws, wf = _guarded(nws)
        n_out = 9 + 3 if grad else 8
        out, of = _guarded(n_out)
        if grad:
            dZ, zf = _guarded(M * D)
            dv, df = _guarded(N) if not run_cg else (None, None)
            st = lib.gpk_cglb_elbo_grad(*desc, ops._p(Xd), N, D, D, ops._p(Yd), 1, ops._p(Zd), M, D, 0.3, 1e-6,
                                        ops._p(v), run_cg, 1e-4, 100, 40, ops._p(out), n_out, ops._p(dZ),
                                        None if dv is None else ops._p(dv), ops._p(ws), ops._stream())
        else:
            st = lib.gpk_cglb_elbo(*desc, ops._p(Xd), N, D, D, ops._p(Yd), 1, ops._p(Zd), M, D, 0.3, 1e-6, ops._p(v),
                                   run_cg, 1e-4, 100, 40, ops._p(out), ops._p(ws), ops._stream())
        _lib.check(st, "gpk_cglb_elbo")
        T.cuda.synchronize()
        for full, n in ((vf, N), (wf, nws), (of, n_out)):
            _guard_ok(full, n)
        if grad:
            _guard_ok(zf, M * D)
            if df is not None:
                _guard_ok(df, N)
        vals = out[:8].cpu().numpy()
        if ref is None:
            ref = vals
        else:
            assert np.array_equal(vals, ref)  # the gradient call's forward gives the same bits


def test_more_refusals_and_strided_inputs():
    X, Y, Z = _reg(60, 6)
    per = gpf.kernels.Periodic(gpf.kernels.SquaredExponential())
    with pytest.raises(NotImplementedError):
        gpf.models.CGLB((X, Y), kernel=per, inducing_variable=Z).elbo()
    lik = gpf.likelihoods.Gaussian(variance=gpf.mean_functions.Linear(A=np.array([[0.05], [0.0]]), b=np.array([0.3])))
    m = gpf.models.CGLB((X, Y), kernel=gpf.kernels.SquaredExponential(), inducing_variable=Z, likelihood=lik)
    with pytest.raises(NotImplementedError, match="constant"):
        m.elbo()
    # gpk_kmv with ldx > D (X a column slice of a wider array)
    rng = np.random.default_rng(0)
    W = rng.standard_normal((300, 5))
    V = rng.standard_normal((300, 2))
    kg = gpf.kernels.SquaredExponential(lengthscales=1.3)
    desc = gpf.kernels.compile_kernel(kg, 3)
    T = _T()
    lib = _lib.load()
    Wd, Vd = T.from_numpy(W).cuda(), T.from_numpy(V).cuda()
    out = T.empty((300, 2), dtype=T.float64, device="cuda")
    ws = ops.scratch_bytes(lib.gpk_kmv_ws(300, 300, 2))
    _lib.check(lib.gpk_kmv(*desc, ops._p(Wd), 300, 5, None, 300, 5, 3, ops._p(Vd), 2, 2, 0.2, ops._p(out), 2,
                           ops._p(ws), ops._stream()), "gpk_kmv")
    ko = O.SquaredExponential(1.0, 1.3)
    ref = (ko.K(W[:, :3]) + 0.2 * np.eye(300)) @ V
    np.testing.assert_allclose(out.cpu().numpy(), ref, rtol=1e-12, atol=1e-12)


# ---- the gradient against the parameter-gradient oracle ----------------------------------------------------------
# |device - oracle| <= C x S per kernel slot and per element of the noise, Z, v and the mean's A and b, S the oracle's
# sum of |terms| (abs_sums), as in tests/test_gpu_grad_dispatch.py (C_CGLB there, where the reasoning is; these cases
# have no sqrt-type leaf).  Measured on an H100 80GB HBM3 (700 W limit): at most 3.1e-14 S at N = 347 (P = 8) and
# 8.3e-15 S in CG mode.
C_GRAD = 1e-11
# At N = 16411 the rounding of z = Q^-1 r is larger by the conditioning of Q ~ N var / s, about 40 times that of the
# N < 500 cases: measured 3.3e-11 S (ARD RBF) and 6.9e-11 S (Matern52 + Linear) on the same H100.
C_GRAD_AT_SIZE = 5e-10
JIT = 1e-6


def _slot_refs(kg, D, g):
    """{Parameter: (oracle gradient, S)} of the kernel slots, from the oracle's per-leaf dicts in slot order."""
    ref = np.concatenate([np.ravel(np.asarray(x, dtype=np.float64)) for gd in g["leaves"] for x in gd.values()])
    sc = np.concatenate([np.ravel(np.asarray(x, dtype=np.float64)) for gd in g["leaves_abs"] for x in gd.values()])
    out = {}
    for p, off, cnt in gpf.kernels.gradient_slots(kg, D):
        out[p] = (ref[off:off + cnt].reshape(p.shape), sc[off:off + cnt].reshape(p.shape))
    assert off + cnt == ref.size
    return out


def _ratio(dev, ref, sc, what, c=C_GRAD):
    dev = np.asarray(dev, dtype=np.float64).reshape(np.shape(ref))
    assert np.all(np.isfinite(dev)), what
    assert not np.any((dev == 0.0) & (ref != 0.0)), f"{what}: an entry is exactly 0 where the oracle's is not"
    return float(np.max(np.abs(dev - ref) / (c * sc)))


def _model_error(m, kg, D, grads, g, mf=None, c=C_GRAD):
    """max |device - oracle| / (C S) over every gradient the model returns."""
    refs = _slot_refs(kg, D, g)
    refs[m.likelihood.variance] = (np.asarray(g["noise_variance"]), np.asarray(g["noise_abs"]))
    refs[m.inducing_variable.Z] = (g["Z"], g["Z_abs"])
    if m.aux_vec.trainable:
        refs[m.aux_vec] = (g["v"], g["v_abs"])
    if mf is not None:
        refs[mf.A] = (g["mean"]["A"], g["mean_abs"]["A"])
        refs[mf.b] = (g["mean"]["b"], g["mean_abs"]["b"])
    assert set(grads) == set(refs)
    return max(_ratio(H.to_np(v) if hasattr(v, "cpu") else v, *refs[p], getattr(p, "name", "?"), c)
               for p, v in grads.items())


def _several_outputs(P):
    rng = np.random.default_rng(40 + P)
    N, M, D = 347, 37, 3
    X = rng.standard_normal((N, D))
    Y = np.sin(X @ rng.standard_normal((D, P))) + 0.2 * rng.standard_normal((N, P))
    Z = rng.standard_normal((M, D))
    v = 0.3 * rng.standard_normal((P, N))
    A, b = 0.1 * rng.standard_normal((D, P)), 0.2 + 0.1 * np.arange(P)
    return X, Y, Z, v, A, b


@pytest.mark.parametrize("P", [1, 2, 3, 8])
def test_gradient_several_outputs_against_oracle(P):
    """Trainable v [P, N] and a Linear mean with A [D, P]: every element of the kernel slots, the noise, Z, v, A and b
    against the oracle, through the model and through gpk_cglb_elbo_grad called directly with guarded buffers (the
    mean's gradient read back from dF/dm in the workspace)."""
    X, Y, Z, v, A, b = _several_outputs(P)
    N, D = X.shape
    M = Z.shape[0]
    s = 0.3
    kg, ko = _pair(("sum", "rbf_ard", "lin"), D)
    ref_val, g = CGO.cglb_elbo_and_grad_expr(X, Y, ko, Z, s, v, mean_function=O.LinearMean(A, b), jitter=JIT,
                                             abs_sums=True)
    mf = gpf.mean_functions.Linear(A=A.copy(), b=b.copy())
    m = gpf.models.CGLB((X, Y), kernel=kg, inducing_variable=Z.copy(), noise_variance=s, mean_function=mf,
                        v_grad_optimization=True)
    m.aux_vec.assign(v.copy())
    val, grads = m.elbo_and_grad()
    np.testing.assert_allclose(float(val), ref_val, rtol=1e-8)
    err_model = _model_error(m, kg, D, grads, g, mf)

    T = _T()
    lib = _lib.load()
    desc = gpf.kernels.compile_kernel(kg, D)
    n_slots = lib.gpk_gpr_lml_grad_slots(*desc, D)
    Yc = Y - (X @ A + b)
    Xd, Yd, Zd = (T.from_numpy(np.ascontiguousarray(a)).cuda() for a in (X, Yc, Z))
    vd = T.from_numpy(v.copy()).cuda()
    n_out = 9 + n_slots
    nws = (lib.gpk_cglb_elbo_grad_ws(N, M, P) + 7) // 8
    dm_off = lib.gpk_cglb_elbo_grad_dm(N, M, P) // 8
    out, of = _guarded(n_out)
    dZ, zf = _guarded(M * D)
    dv, df = _guarded(P * N)
    ws, wf = _guarded(nws)
    _lib.check(lib.gpk_cglb_elbo_grad(*desc, ops._p(Xd), N, D, D, ops._p(Yd), P, ops._p(Zd), M, D, s, JIT, ops._p(vd), 0,
                                      1.0, 100, 40, ops._p(out), n_out, ops._p(dZ), ops._p(dv), ops._p(ws),
                                      ops._stream()), "gpk_cglb_elbo_grad")
    T.cuda.synchronize()
    for full, n in ((of, n_out), (zf, M * D), (df, P * N), (wf, nws)):
        _guard_ok(full, n)
    assert np.array_equal(vd.cpu().numpy(), v)  # no CG: v is read only
    o = out.cpu().numpy()
    np.testing.assert_allclose(o[0], ref_val, rtol=1e-8)
    refs = _slot_refs(kg, D, g)
    slots = np.concatenate([np.ravel(refs[p][0]) for p, _, _ in gpf.kernels.gradient_slots(kg, D)])
    slots_abs = np.concatenate([np.ravel(refs[p][1]) for p, _, _ in gpf.kernels.gradient_slots(kg, D)])
    dm = ws[dm_off:dm_off + N * P].cpu().numpy().reshape(N, P)
    err_direct = max(_ratio(o[9:], slots, slots_abs, "slots"), _ratio(o[8], g["noise_variance"], g["noise_abs"], "noise"),
                     _ratio(dZ.cpu().numpy(), g["Z"], g["Z_abs"], "Z"),
                     _ratio(dv.cpu().numpy(), g["v"], g["v_abs"], "v"),
                     _ratio(X.T @ dm, g["mean"]["A"], g["mean_abs"]["A"], "A"),
                     _ratio(dm.sum(0), g["mean"]["b"], g["mean_abs"]["b"], "b"))
    print(f"cglb grad P={P}: worst |device - oracle| / (C S) = {err_model:.3g} (model), {err_direct:.3g} (direct)")
    assert err_model <= 1.0 and err_direct <= 1.0


def test_gradient_in_cg_mode_against_oracle():
    """CG mode (P = 1): the v CG wrote back, read from the parameter, and the whole gradient against the oracle there."""
    X, Y, Z = _reg(613, 29, D=3, seed=21)
    D = X.shape[1]
    kg, ko = _pair(("prod", "m32", "rbf_ard"), D)
    m = gpf.models.CGLB((X, Y), kernel=kg, inducing_variable=Z.copy(), noise_variance=0.2, cg_tolerance=1e-4)
    val, grads = m.elbo_and_grad()
    assert m.cg_iterations() > 0
    v = m.aux_vec.numpy()
    assert np.any(v != 0.0) and m.aux_vec not in grads
    ref_val, g = CGO.cglb_elbo_and_grad_expr(X, Y, ko, Z, 0.2, v, jitter=JIT, abs_sums=True)
    np.testing.assert_allclose(float(val), ref_val, rtol=1e-8)
    err = _model_error(m, kg, D, grads, g)
    print(f"cglb grad CG mode ({m.cg_iterations()} steps): worst |device - oracle| / (C S) = {err:.3g}")
    assert err <= 1.0


@pytest.mark.parametrize("expr", ["rbf_ard", ("sum", "m52", "lin")], ids=str)
def test_gradient_at_size_against_blockwise_oracle(expr):
    """N = 16411 (past 2^14, off the 64 and 32 tile edges): the N x N pass over 33 million lower-triangle elements,
    gpr_grad_kernel<8, true> for the bare ARD RBF on D = 5 and gpr_grad_expr_kernel<8, 0, true> for Matern52 + Linear,
    against the block-wise oracle with the per-slot bar (its constant grown with the conditioning of Q)."""
    N, M, D = 16411, 61, 5
    rng = np.random.default_rng(5)
    X = rng.standard_normal((N, D))
    Y = np.sin(X[:, :1]) + 0.1 * rng.standard_normal((N, 1))
    Z = rng.standard_normal((M, D))
    v = 0.3 * rng.standard_normal((1, N))
    kg, ko = _pair(expr, D)
    m = gpf.models.CGLB((X, Y), kernel=kg, inducing_variable=Z.copy(), noise_variance=0.15, v_grad_optimization=True)
    m.aux_vec.assign(v.copy())
    val, grads = m.elbo_and_grad()
    t0, w0 = time.process_time(), time.perf_counter()
    ref_val, g = CGO.cglb_elbo_and_grad_expr(X, Y, ko, Z, 0.15, v, jitter=JIT, abs_sums=True)
    cpu, wall = time.process_time() - t0, time.perf_counter() - w0
    np.testing.assert_allclose(float(val), ref_val, rtol=1e-8)
    err = _model_error(m, kg, D, grads, g, c=C_GRAD_AT_SIZE)
    print(f"cglb grad N={N} {expr}: worst |device - oracle| / (C S) = {err:.3g}; oracle {wall:.1f} s wall, {cpu:.1f} s CPU")
    assert err <= 1.0
