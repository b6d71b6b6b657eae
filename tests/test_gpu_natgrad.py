"""Natural-gradient steps on the device (gpk_natgrad_step: csrc/natgrad.cu; gpflow_b200.optimizers.NaturalGradient):
the step against the NumPy oracle (tests/natgrad_oracle.py, pinned against the reference's literal conversions in
tests/test_oracle_natgrad.py) across the factorisation's leaf and int8 engines, the reference's equivalences (VGP and
SVGP reach GPR and SGPR in one XiNat step of size 1; XiSqrtMeanVar gets there in small steps), convergence with the
Bernoulli likelihood and the MultiClass comparison with L-BFGS-B (kernel fixed), minibatches, a failed step, device
residency and the refusals."""
import numpy as np
import pytest

import gpflow_b200 as gpf
from gpflow_b200 import _lib, ops
from gpflow_b200.base import Parameter
from oracle import gp_oracle as O
from tests import natgrad_oracle as NG
from tests.svgp_grad_oracle import _phi, _sym
from tests.test_oracle_natgrad import _grads

pytestmark = pytest.mark.gpu

K, LIK, OPT = gpf.kernels, gpf.likelihoods, gpf.optimizers
XI = {"nat": _lib.GPK_XI_NAT, "sqrt": _lib.GPK_XI_SQRT_MEAN_VAR}


def _device_step(xi, m, S, gm, gS, gamma):
    import torch

    lib = _lib.load()
    M, P = m.shape
    dev = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (m, S, gm, gS)]
    m_out = torch.full_like(dev[0], np.nan)
    S_out = torch.full_like(dev[1], np.nan)
    info = torch.full((P,), 7, dtype=torch.int32, device="cuda")
    ws = ops.scratch_bytes(lib.gpk_natgrad_step_ws(M, P, XI[xi], _lib.GPK_F64))
    _lib.check(lib.gpk_natgrad_step(XI[xi], M, P, *(ops._p(t) for t in dev), gamma, _lib.GPK_F64, ops._p(m_out),
                                    ops._p(S_out), ops._p(info), ops._p(ws), ops._stream()), "gpk_natgrad_step")
    return m_out.cpu().numpy(), S_out.cpu().numpy(), info.cpu().numpy()


def _q(M, P, kind, rng):
    if kind == "small":   # the reference's test_small_q_sqrt_handeled_correctly
        S = np.tile(1e-3 * np.eye(M)[None], (P, 1, 1))
    else:
        S = np.stack([np.tril(0.3 * rng.standard_normal((M, M)) / np.sqrt(M), -1) + np.diag(0.5 + 0.5 * rng.random(M))
                      for _ in range(P)])
        if kind == "negative":
            S *= np.where(rng.random(M) < 0.4, -1.0, 1.0)[None, None, :]
    return 0.5 * rng.standard_normal((M, P)), S


def _cond_B(S, gS, gamma):
    out = []
    for p in range(S.shape[0]):
        Sp = np.tril(S[p])
        d = np.where(np.diag(Sp) < 0, -1.0, 1.0)
        H = _sym(_phi(Sp.T @ gS[p]))
        ev = np.linalg.eigvalsh(np.eye(len(d)) - 2.0 * gamma * d[:, None] * H * d[None, :])
        out.append(ev[-1] / ev[0])
    return max(out)


@pytest.mark.parametrize("xi", ["nat", "sqrt"])
@pytest.mark.parametrize("kind", ["well", "small", "negative"])
@pytest.mark.parametrize("M,P", [(1, 8), (2, 3), (127, 8), (128, 3), (129, 8), (511, 3), (512, 3), (700, 1),
                                 (2048, 1)])
def test_step_matches_the_oracle(cuda_device, xi, kind, M, P):
    rng = np.random.default_rng(1000 * M + P)
    m, S = _q(M, P, kind, rng)
    gm, gS = _grads(M, P, S, rng)
    S_in = S + np.triu(np.full((M, M), np.nan), 1)[None]   # the strict upper part is never read
    for gamma in (1.0, 0.1):
        mr, Sr = NG.rewritten_step(xi, m, S, gm, gS, gamma)
        md, Sd, info = _device_step(xi, m, S_in, gm, gS, gamma)
        assert (info == 0).all(), info
        if xi == "nat" and M >= 512:   # the factorisation of J B J ran its int8 updates with the 7 planes of the hint
            assert _lib.load().gpk_potrf_last_slices() == 7
        cond = _cond_B(S, gS, gamma) if xi == "nat" else 1.0
        ratio = max(np.abs(md - mr).max() / (1e-10 * cond * np.abs(mr).max()),
                    np.abs(Sd - Sr).max() / (1e-10 * cond * np.abs(Sr).max()))
        print(f"natgrad-ratio xi={xi} kind={kind} M={M} P={P} gamma={gamma} cond={cond:.3g} ratio={ratio:.3g}")
        assert ratio <= 1.0
        upper = np.triu(np.ones((M, M), dtype=bool), 1)
        assert (Sd[:, upper].view(np.int64) == 0).all()   # +0.0, bit for bit


def test_zero_diagonal_and_argument_refusals(cuda_device):
    rng = np.random.default_rng(3)
    m, S = _q(5, 2, "well", rng)
    gm, gS = _grads(5, 2, S, rng)
    S[1, 2, 2] = 0.0
    for xi in XI:
        _, _, info = _device_step(xi, m, S, gm, gS, 0.5)
        assert list(info) == [0, -3], info
    with pytest.raises(ValueError, match="gamma"):
        _device_step("nat", m, S, gm, gS, 0.0)
    lib = _lib.load()
    assert lib.gpk_natgrad_step(0, 5, 2, None, None, None, None, 0.1, _lib.GPK_F32, None, None, None, None, None) == -1
    assert b"float64" in lib.gpk_last_error()


def _regression(N, seed=0):
    d = O.make_data(seed, N, 2, 1)
    return d["X"], d["Y"]


def _vgp(X, Y, s2=0.1):
    return gpf.models.VGP((X, Y), K.SquaredExponential(variance=1.2, lengthscales=0.7), LIK.Gaussian(s2))


@pytest.mark.parametrize("N,rtol", [(10, 1e-9), (2048, 1e-10)])
def test_vgp_reaches_gpr_in_one_unit_step(cuda_device, N, rtol):
    """natgrad's test_vgp_vs_gpr: one XiNat step of size 1 makes the VGP ELBO the GPR marginal likelihood, at the
    reference's atol 1e-4, and exactly against GPR(kernel + White(jitter)).  At N = 2048 the measured error is 5.8e-12
    relative on an H100 (printed).  What can move it is the Cholesky's int8 trailing updates at n >= 512: the GPR
    reference gets its conditioning hint (1.2 + 0.1) / 0.1 = 13 and takes S = 6 digit planes, which move the factor by
    about 1e-12 cond relative (potrf.cu::pick_slices), about 1.3e-11 here; the bar is 1e-10, a few times that."""
    X, Y = _regression(N)
    m = _vgp(X, Y)
    OPT.NaturalGradient(1.0).minimize(m.training_loss, [(m.q_mu, m.q_sqrt)])
    elbo = float(m.elbo())
    if N == 10:
        g = gpf.models.GPR((X, Y), K.SquaredExponential(variance=1.2, lengthscales=0.7), noise_variance=0.1)
        assert abs(elbo - float(g.log_marginal_likelihood())) <= 1e-4
    jit = gpf.models.GPR((X, Y), K.SquaredExponential(variance=1.2, lengthscales=0.7) +
                         K.White(variance=gpf.config.default_jitter()), noise_variance=0.1)
    ref = float(jit.log_marginal_likelihood())
    print(f"natgrad-vgp-gpr N={N} rel={abs(elbo - ref) / abs(ref):.3g}")
    assert abs(elbo - ref) <= rtol * abs(ref), (elbo, ref)


@pytest.mark.parametrize("whiten", [True, False])
def test_svgp_reaches_sgpr_in_one_unit_step(cuda_device, whiten):
    d = O.make_data(1, 400, 3, 2, M=40)
    X, Y, Z = d["X"], d["Y"], d["Z"]
    kern = K.SquaredExponential(variance=1.1, lengthscales=0.9)
    m = gpf.models.SVGP(kern, LIK.Gaussian(0.2), Z.copy(), num_latent_gps=2, whiten=whiten, num_data=400)
    OPT.NaturalGradient(1.0).minimize(m.training_loss_closure((X, Y)), [(m.q_mu, m.q_sqrt)])
    elbo = float(m.elbo((X, Y)))
    ref = float(gpf.models.SGPR((X, Y), K.SquaredExponential(variance=1.1, lengthscales=0.9), Z.copy(),
                                noise_variance=0.2).elbo())
    assert abs(elbo - ref) <= 1e-9 * abs(ref), (elbo, ref)


def test_xi_sqrt_mean_var_small_steps_reach_gpr(cuda_device):
    X, Y = _regression(10)
    m = _vgp(X, Y)
    opt = OPT.NaturalGradient(0.01, xi_transform=OPT.XiSqrtMeanVar())
    for _ in range(500):
        opt.minimize(m.training_loss, [(m.q_mu, m.q_sqrt)])
    g = gpf.models.GPR((X, Y), K.SquaredExponential(variance=1.2, lengthscales=0.7), noise_variance=0.1)
    assert abs(float(m.elbo()) - float(g.log_marginal_likelihood())) <= 1e-4


def _freeze_all_but_q(m):
    for p in m.trainable_parameters:
        p.trainable = False
    m.q_mu.trainable = m.q_sqrt.trainable = True


def test_bernoulli_natural_gradient_reaches_the_q_only_optimum(cuda_device):
    """Kernel and Z fixed: XiNat with gamma = 1, 40 steps, against L-BFGS-B over (q_mu, q_sqrt) alone."""
    rng = np.random.default_rng(5)
    N, M = 200, 15
    X = rng.standard_normal((N, 1))
    Y = (np.sin(2 * X) + 0.3 * rng.standard_normal((N, 1)) > 0).astype(np.float64)
    data = (X, Y)

    def model():
        m = gpf.models.SVGP(K.SquaredExponential(variance=2.0, lengthscales=0.8), LIK.Bernoulli(), X[:M].copy(),
                            num_data=N)
        _freeze_all_but_q(m)
        return m

    a = model()
    gpf.optimizers.Scipy().minimize(a.training_loss_closure(data), a.trainable_variables,
                                    options={"maxiter": 5000, "gtol": 1e-12, "ftol": 1e-15})
    ref = float(a.elbo(data))
    b = model()
    opt = OPT.NaturalGradient(1.0)
    for _ in range(40):
        opt.minimize(b.training_loss_closure(data), [(b.q_mu, b.q_sqrt)])
    got = float(b.elbo(data))
    print(f"natgrad-bernoulli ref={ref!r} natgrad={got!r}")
    assert abs(got - ref) <= 1e-6 * abs(ref), (got, ref)


def test_multiclass_natural_gradient_against_scipy_at_equal_gradient_evaluations(cuda_device):
    """The 3-class RobustMax classifier of test_gpu_multiclass (kernel and Z fixed, q only).  The RobustMax bound is not
    concave in q, so H = S^T Sigbar S can have eigenvalues above 1 / (2 gamma): from q_sqrt = I the first steps of 0.1
    and 0.05 are too long.  The loop halves gamma on each failed step (which must leave q unchanged, the mirrors
    included) and spends 800 gradient evaluations, failed calls included.  Observed on an H100: the calls 0 and 1 fail,
    gamma settles at 0.025, the ELBO goes from -1216.2 to -267.94 after 143 evaluations and -264.87 after 800.  L-BFGS-B
    over (q_mu, q_sqrt) stops converged after 143 evaluations at -257.91.  The test pins that outcome: natural gradients
    improve the bound but do not match L-BFGS-B here at an equal number of gradient evaluations."""
    rng = np.random.default_rng(21)
    N, M, C = 240, 12, 3
    X = rng.standard_normal((N, 2))
    ang = np.arctan2(X[:, 1], X[:, 0])
    Y = (np.floor((ang + 0.25 * rng.standard_normal(N) + np.pi) / (2 * np.pi / C)).astype(int) % C)[:, None] * 1.0
    data = (X, Y)
    budget = 800

    def model():
        m = gpf.models.SVGP(K.SquaredExponential(variance=1.0, lengthscales=1.0), LIK.MultiClass(C), X[:M].copy(),
                            num_latent_gps=C, whiten=True)
        _freeze_all_but_q(m)
        return m

    a = model()
    elbo0 = float(a.elbo(data))
    gamma, trace, failures = 0.1, [], []
    for call in range(budget):
        mu0, sq0 = a.q_mu.numpy().copy(), a.q_sqrt.numpy().copy()
        mirror = ops.to_device(a.q_sqrt)
        try:
            OPT.NaturalGradient(gamma).minimize(a.training_loss_closure(data), [(a.q_mu, a.q_sqrt)])
        except ops.NonPositiveDefiniteError:
            failures.append((call, gamma))
            assert np.array_equal(a.q_mu.numpy(), mu0) and np.array_equal(a.q_sqrt.numpy(), sq0)
            assert ops.to_device(a.q_sqrt) is mirror
            gamma *= 0.5
        trace.append(float(a.elbo(data)))
    b = model()
    res = gpf.optimizers.Scipy().minimize(b.training_loss_closure(data), b.trainable_variables,
                                          options={"maxfun": budget, "maxiter": budget})
    n = min(int(res.nfev), budget)
    scipy_elbo = float(b.elbo(data))
    print(f"natgrad-multiclass failures(call, gamma)={failures} final_gamma={gamma} elbo0={elbo0!r} "
          f"natgrad@{n}={trace[n - 1]!r} natgrad@{budget}={trace[-1]!r} scipy@{res.nfev}={scipy_elbo!r}")
    assert failures, "a step of 0.1 is expected to be too long for some q along the way"
    assert trace[-1] > elbo0 + 10.0
    assert scipy_elbo >= trace[n - 1]


def test_one_batch_per_minimize_call(cuda_device):
    rng = np.random.default_rng(8)
    X = rng.standard_normal((300, 2))
    Y = np.sin(X[:, :1]) + 0.1 * rng.standard_normal((300, 1))
    draws = [0]

    def batches():
        while True:
            idx = rng.choice(300, 50, replace=False)
            draws[0] += 1
            yield X[idx], Y[idx]

    m = gpf.models.SVGP(K.SquaredExponential(), LIK.Gaussian(0.1), X[:20].copy(), num_data=300)
    closure = m.training_loss_closure(batches())
    opt = OPT.NaturalGradient(0.1)
    for k in range(5):
        opt.minimize(closure, [(m.q_mu, m.q_sqrt)])
        assert draws[0] == k + 1
    assert np.isfinite(float(m.elbo((X, Y))))


def test_failed_step_leaves_the_parameters_untouched(cuda_device):
    X, Y = _regression(30)
    m = _vgp(X, Y)
    m.q_sqrt.assign(np.tile(0.1 * np.eye(30)[None], (1, 1, 1)))
    dev = "cuda:0"
    mu_dev, sq_dev = ops.to_device(m.q_mu), ops.to_device(m.q_sqrt)
    mu_host, sq_host = m.q_mu.numpy().copy(), m.q_sqrt.numpy().copy()
    mu_bits, sq_bits = mu_dev.clone(), sq_dev.clone()
    with pytest.raises(ops.NonPositiveDefiniteError, match="latent 0.*pivot"):
        OPT.NaturalGradient(10.0).minimize(m.training_loss, [(m.q_mu, m.q_sqrt)])
    assert np.array_equal(m.q_mu.numpy(), mu_host) and np.array_equal(m.q_sqrt.numpy(), sq_host)
    assert m.q_mu.device(dev) is mu_dev and m.q_sqrt.device(dev) is sq_dev
    assert (mu_dev == mu_bits).all() and (sq_dev == sq_bits).all()


def test_the_step_output_becomes_the_device_mirror(cuda_device, monkeypatch):
    """The tensor the step wrote is the parameter's device mirror (same object, same storage), its host value equals
    it, and the next evaluation reads it without an upload."""
    X, Y = _regression(40)
    m = _vgp(X, Y)
    written = {}
    orig = Parameter.assign_device

    def record(self, t):
        written[id(self)] = t
        return orig(self, t)

    monkeypatch.setattr(Parameter, "assign_device", record)
    OPT.NaturalGradient(0.5).minimize(m.training_loss, [(m.q_mu, m.q_sqrt, OPT.XiNat())])
    for p in (m.q_mu, m.q_sqrt):
        out = written[id(p)]
        mirror = ops.to_device(p)
        assert mirror is out and mirror.data_ptr() == out.data_ptr()
        assert np.array_equal(mirror.cpu().numpy(), p.numpy())
    ptr = written[id(m.q_sqrt)].data_ptr()
    m.elbo_and_grad()
    assert ops.to_device(m.q_sqrt) is written[id(m.q_sqrt)] and ops.to_device(m.q_sqrt).data_ptr() == ptr


def test_refusals(cuda_device):
    rng = np.random.default_rng(9)
    X = rng.standard_normal((30, 2))
    Y = np.sin(X[:, :1])
    data = (X, Y)
    ng = OPT.NaturalGradient(0.1)
    m = gpf.models.SVGP(K.SquaredExponential(), LIK.Gaussian(0.1), X[:8].copy(), q_diag=True)
    with pytest.raises(NotImplementedError, match="q_diag"):
        ng.minimize(m.training_loss_closure(data), [(m.q_mu, m.q_sqrt)])
    m = gpf.models.SVGP(K.SquaredExponential(), LIK.Gaussian(0.1), X[:8].copy())

    class Custom(OPT.XiTransform):
        pass

    with pytest.raises(NotImplementedError, match="XiNat and XiSqrtMeanVar"):
        ng.minimize(m.training_loss_closure(data), [(m.q_mu, m.q_sqrt, Custom())])
    other = gpf.models.SVGP(K.SquaredExponential(), LIK.Gaussian(0.1), X[:8].copy())
    with pytest.raises(ValueError, match="loss function's model"):
        ng.minimize(m.training_loss_closure(data), [(other.q_mu, other.q_sqrt)])
    with pytest.raises(ValueError, match="listed twice"):
        ng.minimize(m.training_loss_closure(data), [(m.q_mu, m.q_sqrt), (m.q_mu, m.q_sqrt)])
    m.q_mu.prior = LIK.BetaPrior(1.0, 1.0)
    with pytest.raises(NotImplementedError, match="prior"):
        ng.minimize(m.training_loss_closure(data), [(m.q_mu, m.q_sqrt)])
    m.q_mu.prior = None
    with pytest.raises(ValueError, match="training_loss_closure"):
        ng.minimize(lambda: m.training_loss(data), [(m.q_mu, m.q_sqrt)])
    with pytest.raises(ValueError, match="training_loss_closure"):
        ng.minimize(m.training_loss, [(m.q_mu, m.q_sqrt)])
    v = gpf.models.VGP(data, K.SquaredExponential(), LIK.Bernoulli())
    with pytest.raises(NotImplementedError, match="Gaussian likelihood"):
        ng.minimize(v.training_loss, [(v.q_mu, v.q_sqrt)])
    with pytest.raises(ValueError, match="gamma"):
        OPT.NaturalGradient(-1.0)
    with pytest.raises(ValueError, match="empty"):
        ng.minimize(m.training_loss_closure(data), [])
    # models without a variational q and a device gradient, including an empty var_list
    g = gpf.models.GPR(data, K.SquaredExponential(), noise_variance=0.1)
    for vl in ([], [(m.q_mu, m.q_sqrt)]):
        with pytest.raises(NotImplementedError, match="GPR has no variational"):
            ng.minimize(g.training_loss, vl)
    s = gpf.models.SGPR(data, K.SquaredExponential(), X[:8].copy(), noise_variance=0.1)
    with pytest.raises(NotImplementedError, match="SGPR has no variational"):
        ng.minimize(s.training_loss_closure(), [])
    # SVGP's own device-gradient refusals propagate unchanged: materialised and multi-output kernels
    for kern, cls in [(K.Cosine() + K.White(), "Cosine"), (K.Periodic(K.SquaredExponential()), "Periodic")]:
        mk = gpf.models.SVGP(kern, LIK.Gaussian(0.1), X[:8].copy(), num_latent_gps=1)
        with pytest.raises(NotImplementedError, match=cls):
            ng.minimize(mk.training_loss_closure(data), [(mk.q_mu, mk.q_sqrt)])
    mo = gpf.models.SVGP(K.SharedIndependent(K.SquaredExponential(), 1), LIK.Gaussian(0.1), X[:8].copy(),
                         num_latent_gps=1)
    with pytest.raises(NotImplementedError, match="single-output"):
        ng.minimize(mo.training_loss_closure(data), [(mo.q_mu, mo.q_sqrt)])
    from dataclasses import replace

    with gpf.config.as_context(replace(gpf.config.config(), float=np.float32)):
        m32 = gpf.models.SVGP(K.SquaredExponential(), LIK.Gaussian(0.1), X[:8].copy())
    with pytest.raises(NotImplementedError, match="float64"):
        ng.minimize(m32.training_loss_closure(data), [(m32.q_mu, m32.q_sqrt)])
