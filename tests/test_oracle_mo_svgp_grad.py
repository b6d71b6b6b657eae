"""The SVGP gradient oracle (tests/svgp_grad_oracle.py) with several kernels, inducing sets or W against central finite
differences of its ELBO (composed from O.mo_independent_predict_f, O.mix_latent_gp, O.gauss_kl and the likelihood
oracles): every kernel parameter, the likelihood parameter, every entry of each Z_l, q_mu, the lower q_sqrt and W, for
the four rows with a kernel or an inducing set per latent, both whiten and both q_diag settings, a Gaussian and a
Poisson likelihood; and the argument checks of gpk_svgp_mo_elbo_grad.  No device needed."""
import copy
import ctypes

import numpy as np
import pytest

import gpflow_b200 as gpf
from gpflow_b200 import _lib
from oracle import gp_oracle as O
from tests import grad_check as GC
from tests import kernel_grad_oracle as KG
from tests import lik_oracle as LO
from tests import svgp_grad_oracle as S

RNG_SEED = 20261017
L_, P_, B_, M_, D_ = 2, 3, 7, 4, 2

ROWS = ["shared_kernel_separate_z", "separate_kernels_shared_z", "separate_both", "coregionalization"]


def _setup(row, q_diag, lik_name):
    rng = np.random.default_rng(RNG_SEED + ROWS.index(row) + 10 * q_diag)
    X = rng.standard_normal((B_, D_))
    k1 = O.SquaredExponential(1.2, np.array([0.9, 1.6]))
    k2 = O.Matern32(0.8, 1.3) + O.Linear(0.4)
    Zs = [1.2 * rng.standard_normal((M_, D_)) + 0.1 for _ in range(L_)]
    kernels = {"shared_kernel_separate_z": [k1], "separate_kernels_shared_z": [k1, k2]}.get(row, [k1, k2])
    if row == "separate_kernels_shared_z":
        Zs = Zs[:1]
    W = 0.8 * rng.standard_normal((P_, L_)) if row == "coregionalization" else None
    P = P_ if W is not None else L_
    F = np.sin(X[:, :1] @ np.ones((1, P))) + 0.3 * rng.standard_normal((B_, P))
    Y = LO.targets(lik_name, F, rng) if lik_name != "gaussian" else F + 0.1 * rng.standard_normal(F.shape)
    q_mu = 0.5 * rng.standard_normal((M_, L_))
    if q_diag:
        q_sqrt = 0.3 + 0.5 * rng.random((M_, L_))
    else:
        q_sqrt = np.stack([np.tril(0.2 * rng.standard_normal((M_, M_)), -1) + np.diag(0.4 + 0.5 * rng.random(M_))
                           for _ in range(L_)])
    lik = LO.make(lik_name, **({"variance": 0.3} if lik_name == "gaussian" else {}))
    return X, Y, Zs, kernels, q_mu, q_sqrt, W, lik


@pytest.mark.parametrize("row", ROWS)
@pytest.mark.parametrize("whiten", [True, False])
@pytest.mark.parametrize("q_diag", [False, True])
@pytest.mark.parametrize("lik_name", ["gaussian", "poisson"])
def test_mo_svgp_gradient_matches_finite_differences(row, whiten, q_diag, lik_name):
    X, Y, Zs, kernels, q_mu, q_sqrt, W, lik = _setup(row, q_diag, lik_name)
    h, tol = 1e-5, 5e-6
    num_data = 30

    def f(ks=kernels, zs=Zs, qm=q_mu, qs=q_sqrt, w=W, lk=lik):
        return S.svgp_elbo(X, Y, ks, zs, qm, qs, lk, W=w, whiten=whiten, num_data=num_data)

    elbo, g = S.svgp_elbo_and_grad(X, Y, kernels, Zs, q_mu, q_sqrt, lik, W=W, whiten=whiten, num_data=num_data)
    gk = [g["leaves"]] if len(kernels) == 1 else g["kernels"]
    gz = [g["Z"]] if len(Zs) == 1 else g["Z"]
    assert abs(elbo - f()) < 1e-12 * max(1.0, abs(elbo))
    for ki, k in enumerate(kernels):
        for li, _ in enumerate(KG.leaves(k)):
            for pname, got in gk[ki][li].items():
                for idx in np.ndindex(np.shape(got)):
                    fd = (f(ks=GC.perturb(kernels, li, pname, idx, h, ki))
                          - f(ks=GC.perturb(kernels, li, pname, idx, -h, ki))) / (2 * h)
                    GC.close(float(np.asarray(got)[idx]), fd, tol, (row, ki, li, pname, idx))
    if lik_name == "gaussian":
        fd = (f(lk=LO.Gaussian(0.3 + h)) - f(lk=LO.Gaussian(0.3 - h))) / (2 * h)
        GC.close(g["lik"], fd, tol, "noise")
    else:
        assert g["lik"] == 0.0
    for zi, Z in enumerate(Zs):
        for idx in np.ndindex(Z.shape):
            def fz(v, zi=zi):
                zs = list(Zs)
                zs[zi] = v
                return f(zs=zs)
            GC.close(gz[zi][idx], GC.fd_array(fz, Z, idx, h), tol, ("Z", zi, idx))
    for idx in np.ndindex(q_mu.shape):
        GC.close(g["q_mu"][idx], GC.fd_array(lambda v: f(qm=v), q_mu, idx, h), tol, ("q_mu", idx))
    assert g["q_sqrt"].shape == q_sqrt.shape
    for idx in np.ndindex(q_sqrt.shape):
        if not q_diag and idx[2] > idx[1]:
            assert g["q_sqrt"][idx] == 0.0
            continue
        GC.close(g["q_sqrt"][idx], GC.fd_array(lambda v: f(qs=v), q_sqrt, idx, h), tol, ("q_sqrt", idx))
    if W is None:
        assert g["W"] is None
    else:
        for idx in np.ndindex(W.shape):
            GC.close(g["W"][idx], GC.fd_array(lambda v: f(w=v), W, idx, h), tol, ("W", idx))


def test_mo_oracle_without_mixing_is_the_single_output_oracle_per_latent():
    """SeparateIndependent of L copies of one kernel with a shared Z is the single-output SVGP with P = L."""
    X, Y, Zs, kernels, q_mu, q_sqrt, W, lik = _setup("separate_kernels_shared_z", False, "poisson")
    k = kernels[0]
    e_mo, g_mo = S.svgp_elbo_and_grad(X, Y, [k, copy.deepcopy(k)], Zs, q_mu, q_sqrt, lik, whiten=False, num_data=20)
    e_so, g_so = S.svgp_elbo_and_grad(X, Y, [k], Zs, q_mu, q_sqrt, lik, whiten=False, num_data=20)
    np.testing.assert_allclose(e_mo, e_so, rtol=1e-12)
    for name in g_so["leaves"][0]:
        np.testing.assert_allclose(g_mo["kernels"][0][0][name] + g_mo["kernels"][1][0][name],
                                   g_so["leaves"][0][name], rtol=1e-10)
    for key in ["Z", "q_mu", "q_sqrt"]:
        np.testing.assert_allclose(g_mo[key], g_so[key], rtol=1e-10, atol=1e-12)


# ---- argument checks: status -1 and a readable error, before anything reaches a device ------------------------------
def _call(kernels, D=2, dtype=_lib.GPK_F64, n_out=64, L=2, P=2, n_z=2, W=False, dZ=True, dq_mu=True, dq_sqrt=True,
          dW=True, lik=None):
    lib = _lib.load()
    fake = ctypes.c_void_p(256)  # never dereferenced: every check below runs on the host before the first launch
    lik = lik or _lib.LikDesc(_lib.LIK_GAUSSIAN, 20, 0.0, 0.0, 0.0, 0.1)
    compiled = [gpf.kernels.compile_kernel(k, D) for k in kernels]
    exprs = (_lib.KExpr * len(compiled))(*[_lib.kexpr(c) for c in compiled])
    zp = (ctypes.c_void_p * max(n_z, 1))(*([256] * n_z))
    dzp = (ctypes.c_void_p * max(n_z, 1))(*([256] * n_z))
    st = lib.gpk_svgp_mo_elbo_grad(exprs, len(compiled), fake, 100, D, D, fake, None, P, zp, n_z, 10, D, L, fake, fake,
                                   0, 1, fake if W else None, ctypes.byref(lik), 1.0, 1e-6, dtype, fake, n_out,
                                   dzp if dZ else None, fake if dq_mu else None, fake if dq_sqrt else None,
                                   fake if dW else None, fake, None)
    return st, lib.gpk_last_error().decode()


def test_mo_svgp_grad_entry_point_rejects_bad_arguments():
    K = gpf.kernels
    ks = [K.SquaredExponential(), K.Matern32() + K.Linear()]
    st, msg = _call(ks, dtype=_lib.GPK_F32)
    assert st == -1 and "float64" in msg
    st, msg = _call(ks + [K.Matern52()])           # 3 expressions, L = 2
    assert st == -1 and "n_kernels" in msg
    st, msg = _call(ks, n_z=3)
    assert st == -1 and "n_z" in msg
    st, msg = _call(ks, P=3)                        # no W: P must equal L
    assert st == -1 and "P = 3" in msg and "L = 2" in msg
    st, msg = _call(ks, n_out=9)                    # 5 + 2 + 3 slots needed
    assert st == -1 and "n_out" in msg and "10" in msg
    for missing in ["dZ", "dq_mu", "dq_sqrt"]:
        st, msg = _call(ks, **{missing: False})
        assert st == -1 and "required" in msg and "svgp_mo_elbo_grad" in msg
    st, msg = _call(ks, P=3, W=True, dW=False)
    assert st == -1 and "dW" in msg
    mc = _lib.LikDesc(_lib.LIK_MULTICLASS, 20, 0.0, 0.0, 0.0, 0.0, 1e-3, 3)
    st, msg = _call(ks, lik=mc)                     # MultiClass with 3 classes against P = 2 outputs
    assert st == -1 and "svgp_mo_elbo_grad" in msg
    # the workspace holds one L, A and block-inverse set per latent, and the offset of dF/dm(X) is host arithmetic
    lib = _lib.load()
    gauss = ctypes.byref(_lib.LikDesc(_lib.LIK_GAUSSIAN, 20, 0.0, 0.0, 0.0, 0.1))
    w2 = lib.gpk_svgp_mo_elbo_grad_ws(1000, 64, 2, 3, gauss, _lib.GPK_F64)
    w4 = lib.gpk_svgp_mo_elbo_grad_ws(1000, 64, 4, 3, gauss, _lib.GPK_F64)
    assert w4 - w2 >= 2 * 64 * 1000 * 8
    off = lib.gpk_svgp_mo_elbo_grad_dm(1000, 64, 2, 3, _lib.GPK_F64)
    assert off % 256 == 0 and off + 8 * 1000 * 3 <= w2
