"""Shared pieces of the gradient tests (not collected): the (device kernel, oracle kernel) case table, the inputs the
SVGP / VGP tests feed both sides, central finite differences for the oracle tests and for the device ELBO, and the
comparison of a model's device gradients with an oracle's gradient dict keyed by Parameter."""
import copy
import ctypes

import numpy as np

import gpflow_b200 as gpf
from gpflow_b200 import _lib
from gpflow_b200.base import Exp, Parameter, Shifted, Softplus
from oracle import gp_oracle as O
from tests import hetero_oracle as HO
from tests import kernel_grad_oracle as KG

K = gpf.kernels
ATTRS = ("variance", "lengthscales", "alpha", "offset")
ELL4 = np.array([1.1, 1.9, 0.7, 2.5])


def py_leaves(k):
    """The device kernel's leaves in the order the oracle's `leaves()` numbers them."""
    if isinstance(k, (K.Sum, K.Product)):
        return [leaf for c in k.kernels for leaf in py_leaves(c)]
    return [k]


def case(name, D):
    """(device kernel, oracle kernel) pairs with the same values."""
    s = float(np.sqrt(D))
    if name == "rbf_plus_white":
        return (K.SquaredExponential(variance=1.3, lengthscales=1.7) + K.White(variance=0.05),
                O.SquaredExponential(1.3, 1.7) + O.White(0.05))
    if name == "c5":
        return ((K.SquaredExponential(variance=1.1, lengthscales=s) + K.Matern32(variance=1.0, lengthscales=2 * s))
                * K.Linear(variance=0.5),
                (O.SquaredExponential(1.1, s) + O.Matern32(1.0, 2 * s)) * O.Linear(0.5))
    if name == "rq":
        return (K.RationalQuadratic(variance=1.2, lengthscales=1.6, alpha=0.8), O.RationalQuadratic(1.2, 1.6, alpha=0.8))
    if name == "rq_ard":
        return (K.RationalQuadratic(variance=1.2, lengthscales=ELL4, alpha=2.5), O.RationalQuadratic(1.2, ELL4, alpha=2.5))
    if name == "polynomial_ard":
        v = np.array([0.2, 0.1, 0.3, 0.25])
        return (K.Polynomial(degree=2.0, variance=v, offset=1.3) + K.White(variance=0.1),
                O.Polynomial(degree=2.0, variance=v, offset=1.3) + O.White(0.1))
    if name == "linear_ard":
        v = np.array([0.3, 0.5, 0.9, 0.2])
        return (K.Linear(variance=v) + K.Matern12(variance=0.5, lengthscales=1.5),
                O.Linear(v) + O.Matern12(0.5, 1.5))
    if name == "constant_times_matern52":
        return (K.Constant(variance=1.7) * K.Matern52(variance=0.9, lengthscales=1.8),
                O.Constant(1.7) * O.Matern52(0.9, 1.8))
    if name == "additive_active_dims":
        v = np.array([0.3, 0.4])
        return (K.SquaredExponential(lengthscales=0.9, active_dims=[0]) + K.Matern52(variance=0.7, lengthscales=1.3,
                                                                                    active_dims=[1])
                + K.Exponential(variance=0.4, lengthscales=np.array([1.2, 0.8]), active_dims=[2, 3])
                + K.Linear(variance=v, active_dims=[2, 3]),
                O.SquaredExponential(1.0, 0.9, active_dims=[0]) + O.Matern52(0.7, 1.3, active_dims=[1])
                + O.Exponential(0.4, np.array([1.2, 0.8]), active_dims=[2, 3]) + O.Linear(v, active_dims=[2, 3]))
    if name == "k_plus_k":
        kp = K.Matern32(variance=0.9, lengthscales=ELL4)
        ko = O.Matern32(0.9, ELL4)
        return kp + kp, ko + ko
    raise ValueError(name)


def latent_kernel_pairs(D):
    """Three latent kernels with different slot counts: ARD RBF (1 + D), Matern32 + Linear (3), RationalQuadratic (3)."""
    ell = 0.9 + 0.3 * np.arange(D)
    return ([K.SquaredExponential(variance=1.2, lengthscales=ell), K.Matern32(variance=0.8, lengthscales=1.3)
             + K.Linear(variance=0.4), K.RationalQuadratic(variance=1.1, lengthscales=0.7, alpha=2.0)],
            [O.SquaredExponential(1.2, ell.copy()), O.Matern32(0.8, 1.3) + O.Linear(0.4),
             O.RationalQuadratic(1.1, 0.7, alpha=2.0)])


def hetero_pair(name="exp", lower=0.0):
    """(device HeteroskedasticTFPConditional, oracle) with the scale transform `name` shifted by `lower`."""
    base = Exp() if name == "exp" else Softplus()
    transform = Shifted(base, lower) if lower else base
    return gpf.likelihoods.HeteroskedasticTFPConditional(scale_transform=transform), HO.Hetero(name, lower)


class Datum:  # tests/integration/test_method_equivalence.py:33-40
    rng = np.random.RandomState(0)
    X = rng.rand(20, 1) * 10
    Y = np.sin(X) + 0.9 * np.cos(X * 1.6) + rng.randn(*X.shape) * 0.8
    Y = np.tile(Y, 2)  # two identical columns
    Xtest = rng.rand(10, 1) * 10


def wide_cases():
    """The widest stagings the device gradient takes (tests/test_gpu_grad_dispatch.py): 12 leaves with 36 scalar slots
    in 4 gram groups on D = 10, and 4 gram groups of 32 staged columns on D = 32, three of them ARD."""
    g4 = [None, [0, 1, 2, 3, 4], [5, 6, 7, 8, 9], [9, 0, 3]]
    rq = [O.RationalQuadratic(0.25 + 0.05 * i, (1.2 + 0.25 * i) * (1.6 if g4[i % 4] is None else 1.0),
                              alpha=0.4 + 0.1 * i, active_dims=g4[i % 4]) for i in range(12)]
    rq12 = O.Sum([O.Product(rq[:2]), *rq[2:6], O.Product(rq[6:8]), *rq[8:]])
    ard = O.Sum([O.SquaredExponential(0.9, np.linspace(2.5, 4.5, 10), active_dims=list(range(10))),
                 O.Product([O.Linear(np.linspace(0.05, 0.2, 8), active_dims=list(range(10, 18))),
                            O.Matern32(0.8, 3.0, active_dims=list(range(18, 26)))]),
                 O.RationalQuadratic(0.6, np.linspace(2.0, 3.5, 6), alpha=1.3, active_dims=list(range(26, 32)))])
    return {"rq12_36_slots": (rq12, 10), "ard_4_groups_d32": (ard, 32)}


# ---- inputs ----------------------------------------------------------------------------------------------------------
def z(M, D, seed=3):
    return 1.1 * np.random.default_rng(seed).standard_normal((M, D))


def q(M, P, q_diag=False, seed=4, upper_noise=True):
    """q_mu [M, P] and q_sqrt ([P, M, M], or [M, P] with q_diag), drawn from `seed` (an int or a Generator to draw on).
    With `upper_noise` the strict upper triangle of q_sqrt holds noise that the device must never read; otherwise it is
    zero."""
    rng = np.random.default_rng(seed)
    q_mu = 0.3 * rng.standard_normal((M, P))
    if q_diag:
        return q_mu, 0.4 + 0.6 * rng.random((M, P))
    q_sqrt = np.stack([np.tril(0.1 * rng.standard_normal((M, M)), -1) + np.diag(0.5 + 0.5 * rng.random(M))
                       for _ in range(P)])
    return q_mu, q_sqrt + np.triu(rng.standard_normal((M, M)), 1)[None] if upper_noise else q_sqrt


# ---- finite differences ----------------------------------------------------------------------------------------------
def close(got, fd, tol, what):
    assert abs(got - fd) <= tol * max(1.0, abs(fd)), (what, got, fd)


def fd_array(f, arr, idx, h):
    p, m = arr.copy(), arr.copy()
    p[idx] += h
    m[idx] -= h
    return (f(p) - f(m)) / (2 * h)


def perturb(kernel, leaf, name, idx, h, ki=None):
    """A deep copy of the oracle kernel (or, with `ki`, of the list of kernels, moving kernel ki) with parameter `name`
    of leaf `leaf` moved by h at idx.  A shared leaf (k + k) stays one object after deepcopy: both occurrences move."""
    out = copy.deepcopy(kernel)
    target = KG.leaves(out if ki is None else out[ki])[leaf]
    v = np.array(getattr(target, name), dtype=np.float64)
    if v.ndim == 0:
        v = v + h
    else:
        v = v.copy()
        v[idx] += h
    setattr(target, name, v if v.ndim else float(v))
    return out


def fd_along(m, data, params, dirs, t):
    """Central difference of the device ELBO m.elbo(data) along the directions `dirs` of `params`."""
    base = [np.array(p.numpy(), dtype=np.float64) for p in params]

    def at(s):
        for p, b0, dv in zip(params, base, dirs):
            p.assign(b0 + s * dv)
        return float(m.elbo(data))

    fp, fm = at(t), at(-t)
    at(0.0)
    return (fp - fm) / (2 * t)


# ---- argument checks ------------------------------------------------------------------------------------------------
def svgp_grad_status(nodes, n, dims, ard, D, lik, dtype=_lib.GPK_F64, n_out=64, dZ=True):
    """gpk_svgp_elbo_grad with placeholder pointers and the descriptor `lik`: (status, last error).  Only for the
    argument checks, which return before any device work."""
    lib = _lib.load()
    fake = ctypes.c_void_p(256)
    st = lib.gpk_svgp_elbo_grad(nodes, n, dims, ard, fake, 100, D, D, fake, None, 1, fake, 10, D, fake, fake, 0, 1,
                                ctypes.byref(lik), 1.0, 1e-6, dtype, fake, n_out, fake if dZ else None, fake, fake, fake,
                                None)
    return st, lib.gpk_last_error().decode()


# ---- device against oracle -------------------------------------------------------------------------------------------
def leaf_grads_by_param(kernel, per_leaf):
    """{id(Parameter): value} from per-leaf oracle dicts in the device's leaf order, summed over the leaves a Parameter
    occurs in."""
    pl = py_leaves(kernel)
    assert len(pl) == len(per_leaf)
    out = {}
    for leaf, gd in zip(pl, per_leaf):
        for a in ATTRS:
            p = getattr(leaf, a, None)
            if isinstance(p, Parameter) and a in gd:
                v = np.asarray(gd[a], dtype=np.float64).reshape(p.shape)
                out[id(p)] = out[id(p)] + v if id(p) in out else v
    return out


def reference_by_param(g, kernels, mean_function=None, extra=()):
    """An oracle gradient dict as {id(Parameter): array}: the leaves of each device kernel in `kernels` (g["leaves"] for
    one, g["kernels"] for several; a Parameter shared across kernels sums), the mean function's parameters, and each
    (Parameter, value) of `extra`."""
    per_kernel = [g["leaves"]] if "leaves" in g else g["kernels"]
    assert len(per_kernel) == len(kernels)
    ref = {}
    for kp, gk in zip(kernels, per_kernel):
        for pid, v in leaf_grads_by_param(kp, gk).items():
            ref[pid] = ref[pid] + v if pid in ref else v
    for name, v in g["mean"].items():
        ref[id(getattr(mean_function, name))] = np.asarray(v).reshape(getattr(mean_function, name).shape)
    for p, v in extra:
        ref[id(p)] = np.asarray(v)
    return ref


def assert_grads_match(grads, ref, rtol, rule):
    """The device gradients {Parameter: array} against `ref` from reference_by_param: the same Parameters, every entry
    finite, and |device - oracle| <= atol per Parameter, with atol = rtol x the largest oracle entry of the model
    (rule "model") or rtol x max(the Parameter's largest oracle entry, 1e-3 x the model's) (rule "parameter")."""
    assert {id(p) for p in grads} == set(ref)
    scale = max(float(np.max(np.abs(v))) for v in ref.values())
    for p, g in grads.items():
        g = np.asarray(g, dtype=np.float64).reshape(p.shape)
        assert np.all(np.isfinite(g))
        r = ref[id(p)]
        if rule == "model":
            atol = rtol * scale
        elif rule == "parameter":
            atol = rtol * max(float(np.max(np.abs(r))), 1e-3 * scale)
        else:
            raise ValueError(rule)
        np.testing.assert_allclose(g, r, rtol=0, atol=atol)
