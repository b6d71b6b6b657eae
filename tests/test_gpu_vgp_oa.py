"""VGPOpperArchambeau on the device: the fused value and gradient (gpk_vgp_oa_elbo_grad, csrc/vgp_oa.cu) against the
oracle (tests/vgp_oa_grad_oracle.py, pinned by finite differences in tests/test_oracle_vgp_oa_grad.py) element by
element, for every likelihood; the composed elbo(); finite differences of the device ELBO at N = 2048; the reference's
equivalence with SVGP(whiten=False) and VGP; Scipy and Adam training; predict_f / predict_y / predict_log_density
against a NumPy transcription of vgp.py:379-419; and the refusals.

Tolerances.  Every gradient entry is a sum of products of B_p = A_p^-1 (A_p = I + Lambda_p K Lambda_p), K, alpha,
lambda and the likelihood's adjoints R, W.  A_p's eigenvalues are all >= 1, so ||B_p||_2 <= 1 and
kappa = cond(A_p) <= 1 + max(lambda)^2 ||K||_2.  The factorisation, the inverse chain and the weighted product each
leave a normwise forward error of at most gamma_N kappa (tests/dense64_bounds.py: gamma_k = k u / (1 - k u), plus
the depth of the recursion, which the constant C below covers), so one entry's error is at most
    C gamma_N kappa S_entry,   C = 64,
with S_entry the same sum taken over absolute values (|R| + |W| + 1 and |W| + 1 in place of R and W: fvar's error
reaches R and W through the likelihood's second derivatives, O(1) for these likelihoods).  The oracle's own error is
of the same order and is covered by the same bar."""
import numpy as np
import pytest

import gpflow_b200 as gpf
from gpflow_b200 import ops
from gpflow_b200.models.model import likelihood_scalars
from gpflow_b200.optimizers.adam import _transform_code
from oracle import gp_oracle as O
from tests import adam_oracle as AO
from tests import dense64_bounds as DB
from tests import lik_oracle as LO
from tests import multiclass_oracle as MC
from tests import vgp_oa_grad_oracle as OA
from tests import grad_check as GC
from tests import kernel_grad_oracle as KG

pytestmark = pytest.mark.gpu

K = gpf.kernels
LIK = gpf.likelihoods
C_BAR = 64.0
ELL = np.array([1.3, 0.8, 1.7])


def _kernels(name):
    if name == "ard":   # Sum and Product of fused leaves with ARD lengthscales
        return ((K.SquaredExponential(variance=1.1, lengthscales=ELL) + K.Matern32(variance=0.6, lengthscales=ELL[::-1]))
                * K.Constant(variance=0.9),
                (O.SquaredExponential(1.1, ELL) + O.Matern32(0.6, ELL[::-1].copy())) * O.Constant(0.9))
    v = np.array([0.3, 0.5, 0.2])
    return K.Linear(variance=v), O.Linear(v)


def _liks(name):
    """(device likelihood, oracle likelihood, P or None)."""
    if name == "gaussian":
        return LIK.Gaussian(0.3), LO.Gaussian(0.3), None
    if name == "bernoulli":
        return LIK.Bernoulli(), LO.Bernoulli(), None
    if name == "poisson":
        return LIK.Poisson(), LO.Poisson(), None
    if name == "student_t":
        return LIK.StudentT(scale=0.7, df=4.0), LO.StudentT(0.7, 4.0), None
    if name == "multiclass":
        return LIK.MultiClass(3, invlink=LIK.RobustMax(3, epsilon=0.02)), MC.MultiClass(3, 0.02), 3
    dev, orc = GC.hetero_pair()
    return dev, orc, 2


def _data(lik_name, N, P, seed):
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((N, 3))
    F = np.sin(X[:, :1] + np.arange(P)[None])
    if lik_name == "multiclass":
        Y = MC.labels(rng, F)
    elif lik_name == "hetero":
        Y = F[:, :1] + 0.3 * rng.standard_normal((N, 1))
    else:
        Y = LO.targets(lik_name, F, rng)
    q_alpha = 0.3 * rng.standard_normal((N, P)) / np.sqrt(N)
    q_lambda = 0.6 + rng.random((N, P))
    return X, Y, q_alpha, q_lambda


def _model(X, Y, kp, lik, P, q_alpha, q_lambda, mp=None):
    m = gpf.models.VGPOpperArchambeau((X, Y), kp, lik, mean_function=mp, num_latent_gps=P)
    m.q_alpha.assign(q_alpha)
    m.q_lambda.assign(q_lambda)
    return m


def _bars(X, ko, q_alpha, q_lambda, g, mo):
    """Per-entry error bars C gamma_N kappa S (module docstring), keyed like the oracle's gradient dict."""
    N, P = q_alpha.shape
    _, _, Bs, Kx = OA.moments(X, ko, q_alpha, q_lambda, mo)
    kappa = 1.0 + float(np.max(q_lambda)) ** 2 * float(np.linalg.norm(Kx, 2))
    bar = C_BAR * float(DB.gamma(max(N, 16))) * kappa
    Rt = np.abs(g["R"]) + np.abs(g["W"]) + 1.0
    Wt = np.abs(g["W"]) + 1.0
    aK, aA = np.abs(Kx), np.abs(q_alpha)
    GK = np.zeros((N, N))
    sl = np.empty((N, P))
    for p in range(P):
        lam, aB = q_lambda[:, p], np.abs(Bs[p])
        Abar = aB @ np.diag(Wt[:, p] / lam ** 2 + 0.5) @ aB + 0.5 * aB
        GK += np.outer(Rt[:, p], aA[:, p]) + 0.5 * np.outer(aA[:, p], aA[:, p]) + lam[:, None] * Abar * lam[None]
        sl[:, p] = 2.0 * Wt[:, p] * (1.0 + np.diag(aB)) / lam ** 3 + 2.0 * np.diag(aK @ (lam[:, None] * Abar))
    stacks = []
    KG.walk(ko, np.ones((N, N)), lambda k: k(X), lambda k: KG.leaf_dK(k, X), stacks)
    return {"value": C_BAR * float(DB.gamma(max(N, 16))) * kappa * (2 * N * P + float(np.sum(aA * np.abs(aK @ aA)))),
            "leaves": [{k: bar * np.asarray(v) for k, v in d.items()} for d in KG.reduce(GK, stacks, absolute=True)],
            "lik": bar * (float(np.sum(Rt)) + N * P), "mean": {k: bar * v for k, v in
                                                              KG.mean_grads(mo, np.abs(X), Rt).items()},
            "q_alpha": bar * (aK @ (Rt + aA)), "q_lambda": bar * sl}


def _keyed(m, g, lik_name):
    """Oracle entries keyed by id(Parameter), summed over the leaves a Parameter occurs in."""
    extra = [(m.q_alpha, g["q_alpha"]), (m.q_lambda, g["q_lambda"])]
    extra += [(p, g["lik"]) for p in likelihood_scalars(m.likelihood, 4)]
    return GC.reference_by_param(g, [m.kernel], m.mean_function, extra)


CASES = [  # (likelihood, N, P, kernel, mean function)
    ("gaussian", 1, 1, "ard", None), ("gaussian", 300, 3, "linear", "linear"), ("bernoulli", 37, 3, "ard", "constant"),
    ("bernoulli", 1100, 1, "ard", None), ("poisson", 128, 1, "linear", None), ("poisson", 300, 3, "ard", None),
    ("student_t", 37, 1, "linear", "linear"), ("student_t", 1100, 3, "ard", None), ("multiclass", 37, 3, "ard", None),
    ("multiclass", 300, 3, "linear", None), ("hetero", 128, 2, "ard", None), ("hetero", 1100, 2, "linear", None)]


@pytest.mark.parametrize("lik_name,N,P,kname,mname", CASES)
def test_gradient_matches_oracle_element_by_element(cuda_device, lik_name, N, P, kname, mname):
    dev, orc, Pl = _liks(lik_name)
    P = Pl or P
    X, Y, q_alpha, q_lambda = _data(lik_name, N, P, seed=N + 7 * P)
    kp, ko = _kernels(kname)
    mp = mo = None
    if mname == "linear":
        A, b = 0.2 * np.ones((3, 1)), np.array([0.1])
        mp, mo = gpf.mean_functions.Linear(A=A, b=b), O.LinearMean(A.copy(), b.copy())
    elif mname == "constant":
        mp, mo = gpf.mean_functions.Constant(np.array([0.2])), O.ConstantMean(np.array([0.2]))
    m = _model(X, Y, kp, dev, P, q_alpha, q_lambda, mp)
    elbo, grads = m.elbo_and_grad()
    ref_elbo, g = OA.vgp_oa_elbo_and_grad(X, Y, ko, q_alpha, q_lambda, orc, mean_function=mo)
    bars = _bars(X, ko, q_alpha, q_lambda, g, mo)
    ref, bar = _keyed(m, g, lik_name), _keyed(m, bars, lik_name)
    assert {id(p) for p in grads} == set(ref)
    # the value: log det A_p and tr B_p (N terms each, every one within gamma_N kappa) and alpha^T K alpha
    assert abs(float(elbo) - ref_elbo) <= bars["value"] * (1.0 + abs(ref_elbo))
    np.testing.assert_allclose(float(m.elbo()), float(elbo), rtol=1e-9, atol=1e-9)
    worst = 0.0
    for p, gd in grads.items():
        gd = np.asarray(gd, dtype=np.float64).reshape(p.shape)
        r, b = ref[id(p)], np.maximum(bar[id(p)], 1e-300)
        assert np.all(np.isfinite(gd))
        ratio = np.abs(gd - r) / b
        worst = max(worst, float(np.max(ratio)))
        assert np.all(ratio <= 1.0), (p.name if hasattr(p, "name") else p.shape, float(np.max(ratio)))
    print(f"vgp-oa {lik_name} N={N} P={P} {kname}: worst error / bar = {worst:.3g}")


def test_n2048_finite_difference_of_device_elbo(cuda_device):
    """N = 2048 (a multi-block factorisation on its tensor-core path): the analytic device gradient against central
    finite differences of the composed elbo() along random directions of q_alpha, q_lambda and the lengthscales."""
    N, P = 2048, 1
    X, Y, q_alpha, q_lambda = _data("student_t", N, P, seed=11)
    kp = K.SquaredExponential(variance=1.0, lengthscales=np.array([1.5, 1.2, 1.8])) + K.White(variance=0.05)
    m = _model(X, Y, kp, LIK.StudentT(scale=0.7, df=4.0), P, q_alpha, q_lambda)
    _, grads = m.elbo_and_grad()
    rng = np.random.default_rng(3)
    for p, t in [(m.q_alpha, 1e-3), (m.q_lambda, 1e-4), (kp.kernels[0].lengthscales, 1e-4)]:
        base = np.array(p.numpy(), dtype=np.float64)
        v = rng.standard_normal(base.shape)
        v /= np.linalg.norm(v)

        def at(s):
            p.assign(base + s * v)
            return float(m.elbo())

        fd = (at(t) - at(-t)) / (2 * t)
        p.assign(base)
        got = float(np.sum(np.asarray(grads[p]).reshape(base.shape) * v))
        np.testing.assert_allclose(got, fd, rtol=1e-5, atol=1e-5)


class DatumVGP:  # tests/integration/test_method_equivalence.py (the Opper-Archambeau equivalence data)
    rng = np.random.default_rng(999)
    N, Ns, DX, DY = 10, 10, 2, 2
    X = rng.standard_normal((N, DX))
    Xs = rng.standard_normal((Ns, DX))
    Y = rng.standard_normal((N, DY))
    q_alpha = rng.standard_normal((N, DX))
    q_lambda = rng.standard_normal((N, DX)) ** 2


@pytest.mark.parametrize("lik_name", ["student_t", "gaussian"])
def test_equivalence_with_unwhitened_svgp_and_vgp(cuda_device, lik_name):
    """test_equivalence_vgp_and_opper_archambeau on the device: Matern52; the OA ELBO against SVGP(whiten=False, Z=X)
    at q(u) = N(K alpha, (K^-1 + Lambda^2)^-1) and (Gaussian) against VGP at the whitened q; predict_f as well."""
    d = DatumVGP
    lik = (lambda: LIK.StudentT()) if lik_name == "student_t" else (lambda: LIK.Gaussian(0.5))
    oa = _model(d.X, d.Y, K.Matern52(), lik(), d.DY, d.q_alpha, d.q_lambda)
    Kx = O.Matern52(1.0, 1.0)(d.X) + np.eye(d.N) * gpf.config.default_jitter()
    L = np.linalg.cholesky(Kx)
    L_inv, K_inv = np.linalg.inv(L), np.linalg.inv(Kx)
    mean = Kx @ d.q_alpha
    var = np.linalg.inv(K_inv[None] + np.array([np.diag(l ** 2) for l in d.q_lambda.T]))
    svgp = gpf.models.SVGP(K.Matern52(), lik(), d.X.copy(), num_latent_gps=d.DY, q_mu=mean,
                           q_sqrt=np.linalg.cholesky(var), whiten=False)
    e_oa = float(oa.elbo())
    np.testing.assert_allclose(e_oa, float(svgp.elbo((d.X, d.Y))), rtol=1e-2)
    mu_oa, var_oa = oa.predict_f(d.Xs)
    mu_sv, var_sv = svgp.predict_f(d.Xs)
    np.testing.assert_allclose(mu_oa.cpu().numpy(), mu_sv.cpu().numpy(), rtol=1e-4, atol=1e-10)
    np.testing.assert_allclose(var_oa.cpu().numpy(), var_sv.cpu().numpy(), rtol=1e-4)
    if lik_name == "gaussian":
        vgp = gpf.models.VGP((d.X, d.Y), K.Matern52(), lik(), num_latent_gps=d.DY)
        vgp.q_mu.assign(L_inv @ mean)
        vgp.q_sqrt.assign(np.linalg.cholesky(np.einsum("nN,dNM,mM->dnm", L_inv, var, L_inv)))
        np.testing.assert_allclose(e_oa, float(vgp.elbo()), rtol=1e-2)
        mu_v, var_v = vgp.predict_f(d.Xs)
        np.testing.assert_allclose(mu_oa.cpu().numpy(), mu_v.cpu().numpy(), rtol=1e-4, atol=1e-10)
        np.testing.assert_allclose(var_oa.cpu().numpy(), var_v.cpu().numpy(), rtol=1e-4)


def test_scipy_with_gaussian_reaches_gpr_marginal_likelihood(cuda_device):
    """The OA family holds the exact posterior of a Gaussian likelihood (lambda^2 = 1 / s), so the trained bound reaches
    the GPR log marginal likelihood (the reference's Datum setup)."""
    data = (GC.Datum.X, GC.Datum.Y)
    gpr = gpf.models.GPR(data, kernel=K.SquaredExponential(), mean_function=gpf.mean_functions.Constant())
    oa = gpf.models.VGPOpperArchambeau(data, kernel=K.SquaredExponential(), likelihood=LIK.Gaussian(),
                                       mean_function=gpf.mean_functions.Constant())
    for m in (gpr, oa):
        gpf.optimizers.Scipy().minimize(m.training_loss_closure(), m.trainable_variables, options=dict(maxiter=3000))
    np.testing.assert_allclose(float(oa.maximum_log_likelihood_objective()), float(gpr.log_marginal_likelihood()),
                               rtol=1e-5)
    np.testing.assert_allclose(oa.kernel.lengthscales.numpy(), gpr.kernel.lengthscales.numpy(), rtol=1e-2)


def test_adam_steps_match_oracle_loop(cuda_device):
    """Five device Adam steps on a Bernoulli model against tests/adam_oracle.py driven by the oracle gradient."""
    N, P, steps, lr = 40, 1, 5, 0.05
    X, Y, q_alpha, q_lambda = _data("bernoulli", N, P, seed=5)
    X = X[:, :1]
    m = _model(X, Y, K.SquaredExponential(variance=1.2, lengthscales=0.9), LIK.Bernoulli(), P, q_alpha, q_lambda)
    named = {"variance": m.kernel.variance, "lengthscales": m.kernel.lengthscales, "q_alpha": m.q_alpha,
             "q_lambda": m.q_lambda}
    kinds = {}
    for k, p in named.items():
        code, lower = _transform_code(p)
        kinds[k] = ({gpf._lib.GPK_ADAM_IDENTITY: AO.IDENTITY, gpf._lib.GPK_ADAM_SOFTPLUS: AO.SOFTPLUS,
                     gpf._lib.GPK_ADAM_EXP: AO.EXP}[code], lower)
    value = {k: np.array(p.numpy(), dtype=np.float64) for k, p in named.items()}
    state = {k: (np.zeros_like(v), np.zeros_like(v)) for k, v in value.items()}
    hyper = dict(lr=lr, beta_1=0.9, beta_2=0.999, epsilon=1e-7)
    for t in range(1, steps + 1):
        ko = O.SquaredExponential(float(value["variance"]), float(value["lengthscales"]))
        _, g = OA.vgp_oa_elbo_and_grad(X, Y, ko, value["q_alpha"], value["q_lambda"], LO.Bernoulli())
        grad = {"variance": g["leaves"][0]["variance"], "lengthscales": g["leaves"][0]["lengthscales"],
                "q_alpha": g["q_alpha"], "q_lambda": g["q_lambda"]}
        for k in value:
            gk = np.asarray(grad[k], dtype=np.float64).reshape(value[k].shape)
            value[k], *state[k] = AO.constrained_step(value[k], gk, *state[k], t, *kinds[k], -1.0, **hyper)
    opt = gpf.optimizers.Adam(lr)
    for _ in range(steps):
        opt.minimize(m.training_loss, list(named.values()))
    for k, p in named.items():
        np.testing.assert_allclose(p.numpy(), value[k].reshape(p.shape), rtol=1e-8, atol=1e-10, err_msg=k)


def _predict_ref(X, Xn, ko, q_alpha, q_lambda, full_cov, mo=None):
    """vgp.py:403-419 in NumPy."""
    P = q_alpha.shape[1]
    Kx, Kxx = ko(X, Xn), ko(X)
    mean = Kx.T @ q_alpha + O._mean(mo, Xn, P)
    out = []
    for p in range(P):
        L = np.linalg.cholesky(Kxx + np.diag(1.0 / q_lambda[:, p] ** 2))
        LiKx = np.linalg.solve(L, Kx)
        out.append(ko(Xn) - LiKx.T @ LiKx if full_cov else ko(Xn, full_cov=False) - np.sum(LiKx ** 2, 0))
    return mean, (np.stack(out) if full_cov else np.stack(out, 1))


def test_predictions_match_numpy_transcription(cuda_device):
    N, P = 50, 1
    X, Y, q_alpha, q_lambda = _data("student_t", N, P, seed=9)
    q_alpha *= 10.0
    kp, ko = _kernels("ard")
    A, b = 0.2 * np.ones((3, 1)), np.array([0.1])
    m = _model(X, Y, kp, LIK.StudentT(scale=0.7, df=4.0), P, q_alpha, q_lambda,
               gpf.mean_functions.Linear(A=A, b=b))
    mo = O.LinearMean(A, b)
    Xn = np.random.default_rng(2).standard_normal((13, 3))
    for full_cov in (False, True):
        mu, var = m.predict_f(Xn, full_cov=full_cov)
        rmu, rvar = _predict_ref(X, Xn, ko, q_alpha, q_lambda, full_cov, mo)
        np.testing.assert_allclose(mu.cpu().numpy(), rmu, rtol=1e-9, atol=1e-11)
        np.testing.assert_allclose(var.cpu().numpy(), rvar, rtol=1e-8, atol=1e-10)
    rmu, rvar = _predict_ref(X, Xn, ko, q_alpha, q_lambda, False, mo)
    ym, yv = m.predict_y(Xn)
    em, ev = LO.StudentT(0.7, 4.0).predict_mean_and_var(rmu, rvar)
    np.testing.assert_allclose(ym.cpu().numpy(), em, rtol=1e-8, atol=1e-10)
    np.testing.assert_allclose(yv.cpu().numpy(), ev, rtol=1e-8, atol=1e-10)
    Yn = rmu + 0.3
    ld = m.predict_log_density((Xn, Yn))
    np.testing.assert_allclose(ld.cpu().numpy(), LO.StudentT(0.7, 4.0).predict_log_density(rmu, rvar, Yn), rtol=1e-8)
    with pytest.raises(NotImplementedError):
        m.predict_f(Xn, full_output_cov=True)


class _Quadratic(gpf.mean_functions.MeanFunction):
    def __call__(self, X):
        return ops.to_device(X)[:, :1] * 0.0


def test_refusals(cuda_device):
    d = O.make_data(1, 30, 2, 1)
    data = (d["X"], d["Y"])
    OAM = gpf.models.VGPOpperArchambeau
    with gpf.config.as_context(gpf.config.Config(float=np.float32, jitter=1e-4)):
        m = OAM(data, K.SquaredExponential(), LIK.Gaussian(0.1))
        with pytest.raises(NotImplementedError, match="float64"):
            m.training_loss_and_gradients()
    for kern, cls in [(K.Cosine() + K.White(), "Cosine"), (K.Periodic(K.SquaredExponential()), "Periodic")]:
        with pytest.raises(NotImplementedError, match=cls):
            OAM(data, kern, LIK.Gaussian(0.1)).elbo_and_grad()
    with pytest.raises(NotImplementedError, match="single-output"):
        OAM(data, K.SharedIndependent(K.SquaredExponential(), 1), LIK.Gaussian(0.1)).elbo_and_grad()
    with pytest.raises(NotImplementedError, match="mean function"):
        OAM(data, K.SquaredExponential(), LIK.Gaussian(0.1), mean_function=_Quadratic()).elbo_and_grad()
    lik = LIK.Gaussian(variance=gpf.mean_functions.Linear(A=np.array([[0.05], [0.0]]), b=np.array([0.08])))
    with pytest.raises(NotImplementedError, match="constant variance"):
        OAM(data, K.SquaredExponential(), lik).elbo_and_grad()
    m = OAM(data, K.SquaredExponential(), LIK.Gaussian(0.1))
    m.kernel.variance.prior = object()
    with pytest.raises(NotImplementedError, match="prior"):
        m.elbo_and_grad()
    with pytest.raises(NotImplementedError, match="prior"):
        gpf.optimizers.Scipy().minimize(m.training_loss_closure(), m.trainable_variables, options={"maxiter": 2})
    m = OAM(data, K.SquaredExponential(), LIK.Gaussian(0.1))
    with pytest.raises(NotImplementedError, match="q_mu, q_sqrt"):
        gpf.optimizers.NaturalGradient(0.1).minimize(m.training_loss, [(m.q_alpha, m.q_lambda)])
    with pytest.raises(ValueError, match="latent GPs"):
        OAM((d["X"], d["Y"][:, 0].reshape(-1, 1)), K.SquaredExponential(),
            LIK.MultiClass(3)).elbo_and_grad()
