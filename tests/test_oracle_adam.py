"""The Adam oracle (tests/adam_oracle.py) pinned by hand-computed cases and finite differences, and the host side of
the device optimiser: the lazy host value of base.Parameter, the refusals of optimizers.Adam, its NumPy path against
the oracle, and utilities.training_loop.  No GPU."""
import numpy as np
import pytest

import gpflow_b200 as gpf
from gpflow_b200.base import Module, Parameter, positive, triangular
from gpflow_b200.models.model import LossClosure
from tests import adam_oracle as A

H = A.KERAS_DEFAULTS


def test_first_step_moves_every_coordinate_by_lr_sign_g():
    rng = np.random.default_rng(0)
    g = rng.standard_normal(50) * 10.0 ** rng.integers(-3, 4, 50)
    u0 = rng.standard_normal(50)
    u, m, v = A.adam_step(u0, g, np.zeros(50), np.zeros(50), 1, **H)
    # m_hat = g, sqrt(v_hat) = |g|: the step is lr g / (|g| + epsilon / sqrt(1 - beta_2)), lr sign(g) up to epsilon
    np.testing.assert_allclose(u0 - u, H["lr"] * g / (np.abs(g) + H["epsilon"] / np.sqrt(0.001)), rtol=1e-12)
    big = np.abs(g) > 1.0
    np.testing.assert_allclose((u0 - u)[big], H["lr"] * np.sign(g[big]), rtol=1e-5)
    np.testing.assert_allclose(m, 0.1 * g, rtol=1e-14)
    np.testing.assert_allclose(v, 0.001 * g * g, rtol=1e-12)
    assert A.adam_step(u0, np.zeros(50), np.zeros(50), np.zeros(50), 1, **H)[0].tolist() == u0.tolist()


def test_constant_gradient_keeps_the_step_at_lr():
    u, m, v = np.array([1.0]), np.zeros(1), np.zeros(1)
    for t in range(1, 200):
        new, m, v = A.adam_step(u, np.array([-3.0]), m, v, t, **H)
        # m_hat = g and v_hat = g^2 at every t; epsilon / (|g| sqrt(1 - beta_2^t)) <= 1.06e-6
        np.testing.assert_allclose(new - u, H["lr"], rtol=1.1e-6)
        u = new


def test_bias_correction_values():
    for t, want in [(1, 0.001 * np.sqrt(0.001) / 0.1), (2, 0.001 * np.sqrt(1 - 0.999 ** 2) / (1 - 0.81)),
                    (10, 0.001 * np.sqrt(1 - 0.999 ** 10) / (1 - 0.9 ** 10))]:
        assert A.lr_t(t, 0.001, 0.9, 0.999) == pytest.approx(want, rel=1e-15)
    assert A.lr_t(1, 0.001, 0.9, 0.999) == pytest.approx(3.1622776601683795e-4, rel=1e-12)


def test_one_dimensional_quadratic_by_hand():
    """f(u) = u^2 / 2 from u = 1 with lr = 0.1, beta_1 = 0.5, beta_2 = 0.5, epsilon = 0: two steps written out."""
    h = dict(lr=0.1, beta_1=0.5, beta_2=0.5, epsilon=0.0)
    u1, m1, v1 = A.adam_step(np.array([1.0]), np.array([1.0]), np.zeros(1), np.zeros(1), 1, **h)
    assert (m1[0], v1[0]) == (0.5, 0.5)
    assert u1[0] == pytest.approx(1.0 - 0.1 * np.sqrt(0.5) / 0.5 * 0.5 / np.sqrt(0.5), rel=1e-15)   # = 0.9
    u2, m2, v2 = A.adam_step(u1, u1, m1, v1, 2, **h)
    assert m2[0] == pytest.approx(0.5 + 0.5 * (0.9 - 0.5)) and v2[0] == pytest.approx(0.5 + 0.5 * (0.81 - 0.5))
    assert u2[0] == pytest.approx(0.9 - 0.1 * np.sqrt(0.75) / 0.75 * 0.7 / np.sqrt(0.655), rel=1e-14)


@pytest.mark.parametrize("kind,lower", [(A.SOFTPLUS, 0.0), (A.SOFTPLUS, 1e-6), (A.EXP, 0.0), (A.EXP, 0.3),
                                        (A.IDENTITY, 0.0)])
def test_bijectors_and_chain_rule_against_finite_differences(kind, lower):
    u = np.array([-30.0, -3.0, -0.2, 0.0, 0.7, 4.0, 30.0]) if kind != A.EXP else np.array([-5.0, -0.3, 0.0, 1.2, 4.0])
    y = A.forward(kind, lower, u)
    np.testing.assert_allclose(A.inverse(kind, lower, y), u, rtol=1e-9, atol=1e-9)
    h = 1e-6
    fd = (A.forward(kind, lower, u + h) - A.forward(kind, lower, u - h)) / (2 * h)
    np.testing.assert_allclose(A.forward_grad(kind, u), fd, rtol=1e-7, atol=1e-12)
    # the step through the bijector is the plain step on u with the chain-ruled gradient
    g = np.linspace(-2.0, 3.0, u.size)
    value, m, v = A.constrained_step(y, g, np.zeros_like(u), np.zeros_like(u), 1, kind, lower, -1.0, **H)
    want, _, _ = A.adam_step(A.inverse(kind, lower, y), -g * fd, np.zeros_like(u), np.zeros_like(u), 1, **H)
    np.testing.assert_allclose(A.inverse(kind, lower, value), want, rtol=1e-7, atol=1e-9)


def test_oracle_bijectors_equal_the_package_bijectors():
    y = np.array([1e-3, 0.4, 1.0, 7.0, 40.0])
    for base, kind in (("softplus", A.SOFTPLUS), ("exp", A.EXP)):
        for lower in (0.0, 1e-6):
            t = positive(lower=lower, base=base)
            u = t.inverse(y + lower)
            assert np.array_equal(u, A.inverse(kind, lower, y + lower))
            assert np.array_equal(t.forward(u), A.forward(kind, lower, u))
            assert np.array_equal(t.forward_grad(u), A.forward_grad(kind, u))


class FakeTensor:
    """What Parameter needs of a device tensor, counting the device-to-host copies."""

    class _F64:
        def __str__(self):
            return "torch.float64"

    def __init__(self, arr, device="cuda:0"):
        self.arr, self.device, self.copies = np.array(arr, dtype=np.float64), device, 0
        self.shape, self.dtype = self.arr.shape, self._F64()

    def is_contiguous(self):
        return True

    def detach(self):
        return self

    def cpu(self):
        self.copies += 1
        return self

    def numpy(self):
        return self.arr.copy()


def test_lazy_host_value_state_machine():
    p = Parameter(np.zeros((2, 3)))
    t = FakeTensor(np.arange(6.0).reshape(2, 3))
    p.assign_device(t)
    assert t.copies == 0 and p.shape == (2, 3) and p.dtype == np.float64     # stale: nothing was copied
    assert p._device_cache == {("cuda:0", "float64"): t}
    assert np.array_equal(p.numpy(), t.arr) and t.copies == 1                # the first request fetches
    assert np.array_equal(np.asarray(p), t.arr) and "5." in repr(p) and t.copies == 1   # later ones do not
    t.arr += 1.0                                                             # an optimiser steps in place
    p.device_updated(t)
    assert t.copies == 1
    assert np.array_equal(p.unconstrained_variable, t.arr) and t.copies == 2
    p.device_updated(t)
    p.assign(np.full((2, 3), 7.0))                                           # a host assignment wins
    assert p._device_cache == {} and np.all(p.numpy() == 7.0) and t.copies == 2
    with pytest.raises(ValueError, match="own device mirror"):
        p.device_updated(t)
    with pytest.raises(ValueError, match="contiguous float64 tensor of shape"):
        p.assign_device(FakeTensor(np.zeros((3, 2))))
    q = Parameter(np.eye(3)[None], transform=triangular())
    tq = FakeTensor(2.0 * np.eye(3)[None])
    q.assign_device(tq)
    assert tq.copies == 0 and float(Parameter(5.0)) == 5.0


def test_a_validating_transform_checks_the_device_value_at_once():
    p = Parameter(np.ones(3), transform=positive())
    good, bad = FakeTensor([1.0, 2.0, 3.0]), FakeTensor([1.0, -2.0, 3.0])
    p.assign_device(good)
    assert good.copies == 1 and np.array_equal(p.numpy(), good.arr) and good.copies == 1
    with pytest.raises(ValueError):
        p.assign_device(bad)
    assert np.array_equal(p.numpy(), good.arr) and p._device_cache == {("cuda:0", "float64"): good}
    good.arr[1] = -1.0                      # an in-place update that left the domain is caught when it is read
    p.device_updated(good)
    with pytest.raises(ValueError):
        p.numpy()


def test_constructor_refusals():
    OPT = gpf.optimizers
    with pytest.raises(NotImplementedError, match="amsgrad"):
        OPT.Adam(amsgrad=True)
    with pytest.raises(NotImplementedError, match="schedule"):
        OPT.Adam(learning_rate=lambda step: 0.1)
    with pytest.raises(ValueError, match="beta"):
        OPT.Adam(beta_1=1.0)
    with pytest.raises(ValueError, match="epsilon"):
        OPT.Adam(epsilon=0.0)
    a = OPT.Adam()
    assert (a.learning_rate, a.beta_1, a.beta_2, a.epsilon, a.iterations, a.name) == (0.001, 0.9, 0.999, 1e-7, 0, "Adam")
    with pytest.raises(ValueError, match="training_loss_closure"):
        a.minimize(lambda: 0.0, [])
    with pytest.raises(TypeError, match="Parameter"):
        a.apply_gradients([(np.zeros(2), np.zeros(2))])
    p = Parameter(np.zeros(2))
    with pytest.raises(ValueError, match="twice"):
        a.apply_gradients([(np.zeros(2), p), (np.zeros(2), p)])
    with pytest.raises(NotImplementedError, match="float64"):
        a.apply_gradients([(np.zeros(2), Parameter(np.zeros(2), dtype=np.float32))])
    assert a.iterations == 0


def test_apply_gradients_on_the_host_equals_the_oracle():
    rng = np.random.default_rng(3)
    plain, pos = Parameter(rng.standard_normal((4, 2))), Parameter(0.5 + rng.random(5), transform=positive(lower=1e-6))
    frozen = Parameter(np.ones(2), trainable=False)
    u = [plain.unconstrained_variable.copy(), pos.unconstrained_variable.copy()]
    state = [(np.zeros_like(x), np.zeros_like(x)) for x in u]
    opt = gpf.optimizers.Adam(learning_rate=0.05)
    for t in range(1, 8):
        g = [rng.standard_normal(x.shape) for x in u]
        opt.apply_gradients([(g[0], plain), (g[1], pos), (np.ones(2), frozen)])
        for k in range(2):
            u[k], *state[k] = A.adam_step(u[k], g[k], *state[k], t, lr=0.05, beta_1=0.9, beta_2=0.999, epsilon=1e-7)
        assert opt.iterations == t
    np.testing.assert_allclose(plain.numpy(), u[0], rtol=1e-14)
    np.testing.assert_allclose(pos.unconstrained_variable, u[1], rtol=1e-12)
    assert frozen.numpy().tolist() == [1.0, 1.0]


def test_training_loop_defaults_and_call_count(monkeypatch):
    class Model(Module):
        def __init__(self):
            self.a, self.b = Parameter(1.0), Parameter(2.0, trainable=False)

    model = Model()
    closure = LossClosure(model, lambda: 0.0)
    calls = []
    monkeypatch.setattr(gpf.optimizers.Adam, "minimize",
                        lambda self, loss, var_list: calls.append((self, loss, tuple(var_list))))
    gpf.utilities.training_loop(closure, maxiter=7, compile=True)
    assert len(calls) == 7 and len({id(c[0]) for c in calls}) == 1
    opt = calls[0][0]
    assert isinstance(opt, gpf.optimizers.Adam) and opt.learning_rate == 0.001
    assert all(c[1] is closure and c[2] == (model.a,) for c in calls)
    mine = gpf.optimizers.Adam(0.1)
    gpf.utilities.training_loop(closure, mine, [model.a, model.b], maxiter=2)
    assert [c[0] for c in calls[7:]] == [mine, mine] and calls[-1][2] == (model.a, model.b)
