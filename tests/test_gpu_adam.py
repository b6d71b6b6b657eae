"""Adam on the device (gpk_adam_step: csrc/adam.cu; gpflow_b200.optimizers.Adam): the multi-segment step against the
NumPy oracle (tests/adam_oracle.py, pinned in tests/test_oracle_adam.py) for every bijector, size, alignment and sign;
SVGP training against the oracle-driven loop; VGP, GPR and SGPR against the host loop on the same gradients; minibatches;
the NatGrad + Adam recipe; device residency (no growth of device memory, no host copy of Z, q_mu or q_sqrt) and the
hand-over to Scipy."""
import numpy as np
import pytest

import gpflow_b200 as gpf
from gpflow_b200 import _lib, ops
from gpflow_b200.base import Exp, Parameter, Shifted, Softplus
from oracle import gp_oracle as O
from tests import adam_oracle as A
from tests import grad_check as GC
from tests import lik_oracle as LO

pytestmark = pytest.mark.gpu

K, LIK, OPT = gpf.kernels, gpf.likelihoods, gpf.optimizers
CODE = {A.IDENTITY: _lib.GPK_ADAM_IDENTITY, A.SOFTPLUS: _lib.GPK_ADAM_SOFTPLUS, A.EXP: _lib.GPK_ADAM_EXP}
HYPER = dict(lr=0.01, beta_1=0.9, beta_2=0.999, epsilon=1e-7)


class _Seg:
    """One segment on the device, each array `offset[k]` elements (8 bytes each) into its own allocation, and its
    oracle state."""

    def __init__(self, n, kind, lower, rng, offsets=(0, 0, 0, 0)):
        import torch

        self.n, self.kind, self.lower = n, kind, lower
        value = rng.standard_normal(n) if kind == A.IDENTITY else lower + 0.05 + 3.0 * rng.random(n)
        self.host = [value, rng.standard_normal(n), np.zeros(n), np.zeros(n)]   # value, grad, m, v
        self.dev, self.heads = [], []
        for a, off in zip(self.host, offsets):
            buf = torch.full((n + off,), np.nan, dtype=torch.float64, device="cuda")
            buf[off:] = torch.from_numpy(a)
            self.dev.append(buf[off:])
            self.heads.append(buf[:off])

    def set_grad(self, g):
        import torch

        self.host[1] = g
        self.dev[1].copy_(torch.from_numpy(g))

    def c_seg(self):
        return _lib.AdamSeg(*(t.data_ptr() for t in self.dev), self.n, CODE[self.kind], self.lower)

    def oracle_step(self, t, sign):
        value, g, m, v = self.host
        self.host = [*A.constrained_step(value, g, m, v, t, self.kind, self.lower, sign, **HYPER)]
        self.host.insert(1, g)

    def worst(self):
        """Largest error of value, m, v over the largest magnitude of each."""
        return max(np.abs(self.dev[k].cpu().numpy() - self.host[k]).max() / max(np.abs(self.host[k]).max(), 1e-300)
                   for k in (0, 2, 3)) if self.n else 0.0


def _launch(segs, t, sign):
    arr = (_lib.AdamSeg * len(segs))(*(s.c_seg() for s in segs))
    _lib.check(_lib.load().gpk_adam_step(arr, len(segs), A.lr_t(t, HYPER["lr"], 0.9, 0.999), 0.9, 0.999, 1e-7, sign,
                                         _lib.GPK_F64, ops._stream()), "gpk_adam_step")


KINDS = [(A.IDENTITY, 0.0), (A.SOFTPLUS, 0.0), (A.SOFTPLUS, 1e-6), (A.EXP, 0.0), (A.EXP, 0.25)]


@pytest.mark.parametrize("sign", [1.0, -1.0])
@pytest.mark.parametrize("kind,lower", KINDS)
def test_one_segment_every_size_and_alignment(cuda_device, kind, lower, sign):
    """Offsets: all aligned; all 8 bytes past a 16-byte boundary (the peeled head); value alone misaligned (the
    element-by-element path)."""
    rng = np.random.default_rng(7)
    worst = 0.0
    for n in (1, 2, 3, 4095, 4096, 4097, 2 ** 22 + 1):
        for offsets in ((0, 0, 0, 0), (1, 1, 1, 1), (1, 0, 0, 0)):
            s = _Seg(n, kind, lower, rng, offsets)
            _launch([s], 1, sign)
            s.oracle_step(1, sign)
            worst = max(worst, s.worst())
            assert s.worst() <= 1e-14, (n, offsets, s.worst())
    print(f"adam-kernel kind={kind} lower={lower} sign={sign} worst={worst:.3g}")


@pytest.mark.parametrize("n_segs", [1, 3, 16])
def test_mixed_segments_in_one_launch_over_many_steps(cuda_device, n_segs):
    """Segments of mixed size, bijector and alignment (an empty one included) in one launch; 100 consecutive steps with
    a gradient that changes every step.  One step agrees to 1e-14 of each array's largest magnitude; over 100 steps the
    rounding differences (the device contracts a * b + c into one fused operation, NumPy does not) are carried by the
    moments, and the bar is 1e-12."""
    rng = np.random.default_rng(n_segs)
    sizes = [4097, 1, 0, 33, 2 ** 18 + 3, 2, 700, 5, 4096, 3, 129, 64, 1000, 7, 31, 2 ** 16][:n_segs]
    segs = [_Seg(n, *KINDS[k % len(KINDS)], rng, ((0, 0, 0, 0), (1, 1, 1, 1), (0, 1, 0, 1))[k % 3])
            for k, n in enumerate(sizes)]
    extra = [rng.standard_normal(s.n) for s in segs]
    base = [s.host[1].copy() for s in segs]
    launches = _lib.load().gpk_launch_count
    for t in range(1, 101):
        if t > 1:
            for s, b, e in zip(segs, base, extra):
                s.set_grad(b * np.cos(0.3 * t) + e * np.sin(0.2 * t))
        before = launches()
        _launch(segs, t, -1.0)
        assert launches() - before == 1
        for s in segs:
            s.oracle_step(t, -1.0)
        if t == 1:
            assert max(s.worst() for s in segs) <= 1e-14
    worst = max(s.worst() for s in segs)
    print(f"adam-kernel n_segs={n_segs} steps=100 worst={worst:.3g}")
    assert worst <= 1e-12
    assert all(h.isnan().all() for s in segs for h in s.heads)   # nothing was written before an offset view


def test_argument_refusals(cuda_device):
    lib = _lib.load()
    rng = np.random.default_rng(0)
    s = _Seg(8, A.IDENTITY, 0.0, rng)
    before = [t.clone() for t in s.dev]
    one = (_lib.AdamSeg * 1)(s.c_seg())

    def call(segs=one, n=1, sign=1.0, dtype=_lib.GPK_F64):
        return lib.gpk_adam_step(segs, n, 1e-3, 0.9, 0.999, 1e-7, sign, dtype, ops._stream())

    assert call(dtype=_lib.GPK_F32) == -1 and b"float64" in lib.gpk_last_error()
    assert call(segs=None) == -1
    assert call(n=0) == -1 and call(n=17) == -1 and b"n_segs" in lib.gpk_last_error()
    assert call(sign=0.5) == -1 and b"sign" in lib.gpk_last_error()
    bad = s.c_seg()
    bad.transform = 7
    assert call(segs=(_lib.AdamSeg * 1)(bad)) == -1 and b"transform" in lib.gpk_last_error()
    bad = s.c_seg()
    bad.m = None
    assert call(segs=(_lib.AdamSeg * 1)(bad)) == -1 and b"null" in lib.gpk_last_error()
    bad = s.c_seg()
    bad.n = -1
    assert call(segs=(_lib.AdamSeg * 1)(bad)) == -1
    bad = s.c_seg()
    bad.grad = s.dev[1].data_ptr() + 4
    assert call(segs=(_lib.AdamSeg * 1)(bad)) == -1 and b"aligned" in lib.gpk_last_error()
    assert all((a == b).all() for a, b in zip(before, s.dev))
    assert call() == 0


# ---- models --------------------------------------------------------------------------------------------------------
def _kind(p):
    t, lower = p.transform, 0.0
    if isinstance(t, Shifted):
        t, lower = t.base, t.lower
    return ({Softplus: A.SOFTPLUS, Exp: A.EXP}.get(type(t), A.IDENTITY), lower)


def _named(m):
    out = {"variance": m.kernel.variance, "lengthscales": m.kernel.lengthscales, "Z": m.inducing_variable.Z,
           "q_mu": m.q_mu, "q_sqrt": m.q_sqrt}
    if isinstance(m.likelihood, LIK.Gaussian):
        out["lik"] = m.likelihood.variance
    return out


@pytest.mark.parametrize("M", [17, 64])
@pytest.mark.parametrize("lik", ["gaussian", "bernoulli"])
@pytest.mark.parametrize("whiten,q_diag", [(True, False), (False, False), (True, True), (False, True)])
def test_svgp_minimize_equals_the_oracle_driven_loop(cuda_device, whiten, q_diag, lik, M):
    B, D, P, steps = 120, 3, 2, 30
    d = O.make_data(5, B, D, P)
    X = d["X"]
    Y = d["Y"] if lik == "gaussian" else LO.targets(lik, np.sin(X[:, :1] @ np.ones((1, P))), np.random.default_rng(M))
    q_mu, q_sqrt = GC.q(M, P, q_diag)
    m = gpf.models.SVGP(K.SquaredExponential(variance=1.3, lengthscales=1.7),
                        LIK.Gaussian(0.3) if lik == "gaussian" else LIK.Bernoulli(), GC.z(M, D), num_latent_gps=P,
                        q_mu=q_mu.copy(), q_sqrt=q_sqrt.copy(), whiten=whiten, q_diag=q_diag, num_data=1000)
    named = _named(m)
    assert set(named.values()) == set(m.trainable_variables)
    start = {k: np.array(p.numpy()) for k, p in named.items()}
    want = A.svgp_loop(X, Y, {k: (np.array(p.numpy()), *_kind(p)) for k, p in named.items()}, steps, lik=lik,
                       whiten=whiten, num_data=1000, jitter=gpf.config.default_jitter(), **HYPER)
    opt = OPT.Adam(HYPER["lr"])
    closure = m.training_loss_closure((X, Y))
    for _ in range(steps):
        opt.minimize(closure, m.trainable_variables)
    assert opt.iterations == steps
    worst = 0.0
    for k, p in named.items():
        got = p.numpy()
        assert np.abs(got - start[k]).max() > 1e-3, k
        worst = max(worst, np.abs(got - want[k]).max() / max(1.0, np.abs(want[k]).max()))
    print(f"adam-svgp whiten={whiten} q_diag={q_diag} lik={lik} M={M} worst={worst:.3g}")
    assert worst <= 1e-8   # measured on an H100: 1e-14 .. 4e-14 at M = 17, up to 2.4e-9 at M = 64 (whiten=False)
    if not q_diag:   # the strict upper triangle: zero gradient, zero moments, never written differently
        upper = np.triu(np.ones((M, M), dtype=bool), 1)
        assert np.array_equal(m.q_sqrt.numpy()[:, upper].view(np.int64), q_sqrt[:, upper].view(np.int64))


def _host_loop(m, closure, steps, lr):
    """The loop a user writes on value_and_gradients: host gradients, the oracle's step on the unconstrained variables."""
    variables = m.trainable_variables
    state = [(np.zeros(p.shape), np.zeros(p.shape)) for p in variables]
    for t in range(1, steps + 1):
        _, grads = closure.value_and_gradients(variables)
        for k, (p, g) in enumerate(zip(variables, grads)):
            u, *state[k] = A.adam_step(p.unconstrained_variable, np.asarray(g).reshape(p.shape), *state[k], t,
                                       **{**HYPER, "lr": lr})
            p.assign_unconstrained(u)


def _regression(N, D=2, seed=0):
    d = O.make_data(seed, N, D, 1)
    return d["X"], d["Y"]


@pytest.mark.parametrize("model", ["vgp", "gpr", "sgpr"])
def test_internal_data_models_equal_the_host_loop(cuda_device, model):
    X, Y = _regression(60)

    def make():
        kern = K.SquaredExponential(variance=1.2, lengthscales=0.7) + K.White(variance=0.05)
        if model == "vgp":
            return gpf.models.VGP((X, Y), kern, LIK.Gaussian(0.1), mean_function=gpf.mean_functions.Constant(0.2))
        if model == "gpr":
            return gpf.models.GPR((X, Y), kern, mean_function=gpf.mean_functions.Linear(np.ones((2, 1)), 0.1),
                                  noise_variance=0.1)
        return gpf.models.SGPR((X, Y), kern, X[:9].copy(), noise_variance=0.1)

    a, b = make(), make()
    elbo0 = float(a.maximum_log_likelihood_objective())
    opt = OPT.Adam(0.02)
    for _ in range(25):
        opt.minimize(a.training_loss, a.trainable_variables)
    _host_loop(b, b.training_loss_closure(), 25, 0.02)
    assert float(a.maximum_log_likelihood_objective()) > elbo0
    assert len(a.trainable_variables) == len(b.trainable_variables) >= 4
    for p, q in zip(a.trainable_variables, b.trainable_variables):
        np.testing.assert_allclose(p.numpy(), q.numpy(), rtol=1e-9, atol=1e-9)
    if model == "vgp":
        upper = np.triu(np.ones((60, 60), dtype=bool), 1)
        assert (a.q_sqrt.numpy()[:, upper] == 0.0).all()


def test_apply_gradients_with_device_and_host_gradients(cuda_device):
    """A user's own loop: unconstrained loss gradients, Z's and q_mu's handed over as device tensors."""
    import torch

    X, Y = _regression(80)

    def make():
        return gpf.models.SVGP(K.SquaredExponential(), LIK.Gaussian(0.1), X[:10].copy(), num_data=80)

    a, b = make(), make()
    opt = OPT.Adam(0.01)
    closure = a.training_loss_closure((X, Y))
    for _ in range(5):
        variables = a.trainable_variables
        _, grads = closure.value_and_gradients(variables)
        pairs = [(torch.from_numpy(np.ascontiguousarray(g)).cuda() if p in (a.q_mu, a.inducing_variable.Z) else g, p)
                 for g, p in zip(grads, variables)]
        opt.apply_gradients(pairs)
    _host_loop(b, b.training_loss_closure((X, Y)), 5, 0.01)
    for p, q in zip(a.trainable_variables, b.trainable_variables):
        np.testing.assert_allclose(p.numpy(), q.numpy(), rtol=1e-10, atol=1e-10)


def _batches(X, Y, size, rng, draws):
    while True:
        idx = rng.choice(X.shape[0], size, replace=False)
        draws[0] += 1
        yield X[idx], Y[idx]


def test_one_batch_per_step_and_training_loop(cuda_device):
    rng = np.random.default_rng(8)
    X = rng.standard_normal((300, 2))
    Y = np.sin(X[:, :1]) + 0.1 * rng.standard_normal((300, 1))
    draws = [0]
    m = gpf.models.SVGP(K.SquaredExponential(), LIK.Gaussian(0.1), X[:20].copy(), num_data=300)
    closure = m.training_loss_closure(_batches(X, Y, 50, rng, draws))
    opt = OPT.Adam(0.01)
    for k in range(5):
        opt.minimize(closure, m.trainable_variables)
        assert draws[0] == k + 1
    m.q_mu.prior = LIK.BetaPrior(1.0, 1.0)
    with pytest.raises(NotImplementedError, match="prior"):
        opt.minimize(closure, m.trainable_variables)
    m.q_mu.prior = None
    with pytest.raises(ValueError, match="not a parameter of the model"):
        opt.minimize(closure, [Parameter(1.0)])
    assert draws[0] == 5 and opt.iterations == 5          # a refused call draws no batch
    before = float(m.elbo((X, Y)))
    gpf.utilities.training_loop(closure, maxiter=40)      # Adam(), every trainable variable
    assert draws[0] == 45
    assert float(m.elbo((X, Y))) > before


def test_untrainable_and_unlisted_variables_are_untouched_and_refusals(cuda_device):
    X, Y = _regression(50)
    # away from q = the prior, where the whitened ELBO does not depend on the lengthscale
    m = gpf.models.SVGP(K.SquaredExponential(), LIK.Gaussian(0.1), X[:8].copy(), num_data=50,
                        q_mu=0.3 * np.random.default_rng(1).standard_normal((8, 1)))
    m.kernel.variance.trainable = False
    keep = {p: np.array(p.numpy()) for p in m.parameters}
    OPT.Adam(0.05).minimize(m.training_loss_closure((X, Y)), [m.q_mu, m.kernel.variance, m.kernel.lengthscales])
    changed = {p for p in m.parameters if not np.array_equal(p.numpy(), keep[p])}
    assert changed == {m.q_mu, m.kernel.lengthscales}
    f = gpf.models.GPRFITC((X, Y), K.SquaredExponential(), X[:8].copy(), noise_variance=0.1)
    with pytest.raises(NotImplementedError, match="GPRFITC has no device gradient"):
        OPT.Adam().minimize(f.training_loss_closure(), f.trainable_variables)
    mk = gpf.models.SVGP(K.Cosine() + K.White(), LIK.Gaussian(0.1), X[:8].copy())
    with pytest.raises(NotImplementedError, match="Cosine"):
        OPT.Adam().minimize(mk.training_loss_closure((X, Y)), mk.trainable_variables)


def test_natgrad_plus_adam_recipe_reaches_the_collapsed_bound(cuda_device):
    """The reference's recipe: q_mu and q_sqrt untrainable, one NaturalGradient step (gamma = 1, Gaussian likelihood:
    the optimal q) then one Adam step on the hyperparameters and Z per iteration.  The ELBO rises on average (block
    means of 20 iterations), and after a last natural-gradient step it is SGPR's collapsed bound at the same
    hyperparameters to 1e-7 relative."""
    d = O.make_data(2, 500, 2, 1, M=20)
    X, Y, Z = d["X"], d["Y"], d["Z"]
    m = gpf.models.SVGP(K.SquaredExponential(variance=1.0, lengthscales=1.0), LIK.Gaussian(0.5), Z.copy(), num_data=500)
    gpf.utilities.set_trainable([m.q_mu, m.q_sqrt], False)
    closure = m.training_loss_closure((X, Y))
    natgrad, adam = OPT.NaturalGradient(1.0), OPT.Adam(0.02)
    variables = m.trainable_variables
    assert m.q_mu not in variables and m.inducing_variable.Z in variables
    trace = []
    for _ in range(100):
        natgrad.minimize(closure, [(m.q_mu, m.q_sqrt)])
        adam.minimize(closure, variables)
        trace.append(float(m.elbo((X, Y))))
    blocks = np.mean(np.reshape(trace, (5, 20)), axis=1)
    print(f"adam-recipe block means {blocks}")
    assert (np.diff(blocks) > 0).all()
    natgrad.minimize(closure, [(m.q_mu, m.q_sqrt)])
    ref = gpf.models.SGPR((X, Y), K.SquaredExponential(variance=float(m.kernel.variance.numpy()),
                                                       lengthscales=float(m.kernel.lengthscales.numpy())),
                          m.inducing_variable.Z.numpy().copy(), noise_variance=float(m.likelihood.variance.numpy()))
    got, want = float(m.elbo((X, Y))), float(ref.elbo())
    print(f"adam-recipe elbo={got!r} sgpr={want!r}")
    assert abs(got - want) <= 1e-7 * abs(want)


def test_device_residency_and_the_handover_to_scipy(cuda_device, monkeypatch):
    """During the loop: no growth of allocated device memory between step 2 and step 40, no device-to-host copy of Z,
    q_mu or q_sqrt.  Afterwards numpy() is the mirror, and Scipy starts from Adam's values."""
    import torch

    d = O.make_data(3, 400, 3, 2, M=128)
    X, Y = ops.to_device(d["X"]), ops.to_device(d["Y"])
    m = gpf.models.SVGP(K.SquaredExponential(), LIK.Gaussian(0.2), d["Z"].copy(), num_latent_gps=2, num_data=400)
    big = (m.inducing_variable.Z, m.q_mu, m.q_sqrt)
    start = [np.array(p.numpy()) for p in big]
    fetched = []
    host = Parameter._host
    monkeypatch.setattr(Parameter, "_host",   # records the calls that copy from the device
                        lambda self: (fetched.append(self) if self._newer is not None else None, host(self))[1])
    opt = OPT.Adam(0.01)
    closure = m.training_loss_closure((X, Y))
    mirrors, allocated = None, {}
    for step in range(1, 41):
        opt.minimize(closure, m.trainable_variables)
        if step == 1:
            mirrors = [ops.to_device(p) for p in big]
            fetched.clear()     # the first step uploaded the initial values
        torch.cuda.synchronize()
        allocated[step] = torch.cuda.memory_allocated()
    assert allocated[40] <= allocated[2], allocated
    assert not [p for p in fetched if p in big]
    assert all(ops.to_device(p) is t for p, t in zip(big, mirrors))     # updated in place, never replaced
    for p, t, s in zip(big, mirrors, start):
        assert np.array_equal(p.numpy(), t.cpu().numpy()) and not np.array_equal(p.numpy(), s)
    assert len([p for p in fetched if p in big]) == 3
    monkeypatch.undo()
    x0 = OPT.Scipy.initial_parameters(m.trainable_variables)
    seen = []
    orig = closure.value_and_gradients

    def spy(variables):
        seen.append(OPT.Scipy.initial_parameters(variables))
        return orig(variables)

    closure.value_and_gradients = spy
    loss0 = float(closure())
    OPT.Scipy().minimize(closure, m.trainable_variables, options={"maxiter": 3})
    np.testing.assert_allclose(seen[0], x0, rtol=1e-12, atol=1e-12)
    assert float(closure()) < loss0
