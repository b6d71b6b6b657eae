"""The VGPOpperArchambeau oracle (tests/vgp_oa_grad_oracle.py) against central finite differences of a literal
transcription of gpflow/models/vgp.py:343-376 for every gradient entry (kernel slots, the likelihood's parameter,
q_alpha, q_lambda, the mean function) and every likelihood the device covers; and the identity of the reference's
test_equivalence_vgp_and_opper_archambeau: the OA ELBO is the unwhitened SVGP ELBO at Z = X with q(u) = N(K alpha,
(K^-1 + Lambda^2)^-1).  No device needed."""
import numpy as np
import pytest

from oracle import gp_oracle as O
from tests import grad_check as GC
from tests import hetero_oracle as HO
from tests import kernel_grad_oracle as KG
from tests import lik_oracle as LO
from tests import multiclass_oracle as MC
from tests import svgp_grad_oracle as S
from tests import vgp_oa_grad_oracle as OA

LIKS = ["gaussian", "bernoulli", "poisson", "student_t", "multiclass", "hetero"]


def make_case(lik_name, N=6, D=2, P=None, seed=0):
    """(X, Y, lik oracle, P, q_alpha, q_lambda) with q away from its initial values."""
    rng = np.random.default_rng(20261018 + seed)
    X = rng.standard_normal((N, D))
    if lik_name == "multiclass":
        P = 3
        lik = MC.MultiClass(P, epsilon=0.02)
        Y = MC.labels(rng, np.stack([np.sin(X[:, 0] + c) for c in range(P)], 1))
    elif lik_name == "hetero":
        P = 2
        lik = HO.Hetero("exp")
        Y = np.sin(X[:, :1]) + 0.3 * rng.standard_normal((N, 1))
    else:
        P = P or 2
        lik = LO.make(lik_name, **({"variance": 0.3} if lik_name == "gaussian" else
                                   {"scale": 0.7, "df": 4.0} if lik_name == "student_t" else {}))
        Y = LO.targets(lik_name, np.sin(X[:, :1]) @ np.ones((1, P)), rng)
    q_alpha = 0.4 * rng.standard_normal((N, P))
    q_lambda = 0.6 + rng.random((N, P))
    return X, Y, lik, P, q_alpha, q_lambda


def _lik_param(lik):
    for name in ("variance", "scale", "epsilon"):
        if hasattr(lik, name):
            return name
    return None


@pytest.mark.parametrize("lik_name", LIKS)
def test_oracle_matches_finite_differences_of_the_literal_elbo(lik_name):
    X, Y, lik, P, q_alpha, q_lambda = make_case(lik_name)
    kernel = (O.SquaredExponential(1.1, np.array([1.3, 0.8])) + O.Matern32(0.6, 1.7)) * O.Linear(0.5) + O.White(0.05)
    mf = O.LinearMean(np.full((X.shape[1], 1), 0.2), np.array([0.1]))
    tol, h = 2e-6, 1e-5

    def f(k=kernel, qa=q_alpha, ql=q_lambda, lk=lik):
        return OA.elbo_literal(X, Y, k, qa, ql, lk, mf)

    elbo, g = OA.vgp_oa_elbo_and_grad(X, Y, kernel, q_alpha, q_lambda, lik, mean_function=mf)
    assert abs(elbo - f()) < 1e-12 * max(1.0, abs(elbo))
    for li, leaf in enumerate(KG.leaves(kernel)):
        for pname, val in g["leaves"][li].items():
            for idx in np.ndindex(np.shape(val)):
                fd = (f(k=GC.perturb(kernel, li, pname, idx, h))
                      - f(k=GC.perturb(kernel, li, pname, idx, -h))) / (2 * h)
                GC.close(float(np.asarray(val)[idx]), fd, tol, (li, pname, idx))
    for idx in np.ndindex(q_alpha.shape):
        GC.close(g["q_alpha"][idx], GC.fd_array(lambda v: f(qa=v), q_alpha, idx, h), tol, ("q_alpha", idx))
        GC.close(g["q_lambda"][idx], GC.fd_array(lambda v: f(ql=v), q_lambda, idx, h), tol, ("q_lambda", idx))
    name = _lik_param(lik)
    if name is None:
        assert g["lik"] == 0.0
    else:
        v0 = getattr(lik, name)
        vals = []
        for s in (h, -h):
            setattr(lik, name, v0 + s)
            vals.append(f())
        setattr(lik, name, v0)
        GC.close(g["lik"], (vals[0] - vals[1]) / (2 * h), tol, name)
    for pname, arr in (("A", mf.A), ("b", mf.b)):
        for idx in np.ndindex(arr.shape):
            fd = GC.fd_array(lambda v: _with(mf, pname, v, f), arr, idx, h)
            GC.close(g["mean"][pname][idx], fd, tol, (pname, idx))


def _with(mf, name, value, f):
    old = getattr(mf, name)
    setattr(mf, name, value)
    try:
        return f()
    finally:
        setattr(mf, name, old)


def test_direct_and_diagonal_lambda_forms_agree():
    """The device takes the second term of dF/dlambda from diagonals only: 2 (K Lambda Abar)_jj = 2 [(W_j / lambda_j^2 +
    1/2) B_jj - 1/2 - Abar_jj] / lambda_j, through A Abar = (D + 1/2 I) B - 1/2 I."""
    X, Y, lik, P, q_alpha, q_lambda = make_case("bernoulli", N=9, seed=3)
    kernel = O.Matern52(1.2, 0.9)
    _, fvar, Bs, K = OA.moments(X, kernel, q_alpha, q_lambda)
    _, g = OA.vgp_oa_elbo_and_grad(X, Y, kernel, q_alpha, q_lambda, lik)
    for p in range(P):
        lam, B, W = q_lambda[:, p], Bs[p], g["W"][:, p]
        Abar = B @ np.diag(W / lam ** 2 + 0.5) @ B - 0.5 * B
        diag_form = -2.0 * W * (1.0 - np.diag(B)) / lam ** 3 + 2.0 * (
            (W / lam ** 2 + 0.5) * np.diag(B) - 0.5 - np.diag(Abar)) / lam
        np.testing.assert_allclose(diag_form, g["q_lambda"][:, p], rtol=1e-10, atol=1e-12)


@pytest.mark.parametrize("lik_name", ["gaussian", "student_t", "bernoulli"])
def test_equals_unwhitened_svgp_at_z_equal_x(lik_name):
    """tests/integration/test_method_equivalence.py::test_equivalence_vgp_and_opper_archambeau in NumPy: with Z = X, no
    jitter and q(u) = N(K alpha, (K^-1 + Lambda^2)^-1), the unwhitened SVGP ELBO is the OA ELBO."""
    X, Y, lik, P, q_alpha, q_lambda = make_case(lik_name, N=8, seed=5)
    kernel = O.Matern52(1.3, 1.1)
    K = kernel(X)
    q_mu = K @ q_alpha
    q_sqrt = np.stack([np.linalg.cholesky(np.linalg.inv(np.linalg.inv(K) + np.diag(q_lambda[:, p] ** 2)))
                       for p in range(P)])
    e_oa = OA.elbo_literal(X, Y, kernel, q_alpha, q_lambda, lik)
    e_sv = S.svgp_elbo(X, Y, [kernel], [X], q_mu, q_sqrt, lik, whiten=False, jitter=0.0)
    np.testing.assert_allclose(e_oa, e_sv, rtol=1e-8)
