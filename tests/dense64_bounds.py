"""Error bars and CPU mirrors for the fp64 dense linear algebra under the device gradients, CPU only.

The operators are the tiled GEMM (csrc/gemm.cu), the inverse-based triangular solve (potrf.cu::trsm_rec), the inverse
chain of grad.cu (put_dinv_kernel, trtri_rec, lauum_rec) and fused.cu::chol_adjoint.  References are long double
(64-bit mantissa) products, on sampled rows and columns for large shapes; u = 2^-53, gamma_k = k u / (1 - k u)
(Higham, Accuracy and Stability of Numerical Algorithms, 2nd ed.: ch. 3 for dot products, ch. 8 for triangular
systems, ch. 14 for triangular inverses).  Every bar below assumes only that each floating-point step (multiply, add,
fma, or a DMMA step) is correctly rounded, in whatever order the kernel accumulates.

GEMM.  Each entry of op(A) op(B) is a k-term dot product; whatever the order of its additions (a chain of fmas per k4
step on DMMA, the 8-warp split of the skinny kernel, the column sums of COLSUMSQ), it is within gamma_k of
|op(A)| |op(B)| (Higham (3.5)).  The epilogue rounds alpha * acc, beta * C0 and their sum, so
    |C_dev - C| <= gamma_{k+2} (|alpha| |op(A)| |op(B)| + |beta| |C0|)            elementwise.
The long double reference carries 2^-64 k of the same scale, added to the bar.  COLSUMSQ: the column sum
s_j = sum_i (alpha c_ij)^2 of m rounded squares of entries each within gamma_{k+1}: |s_dev - s| <= (2 gamma_{k+1} +
gamma_{m+1}) sum_i (alpha |op(A)| |op(B)|)_ij^2, plus the accumulation onto the old value (one rounding).

TRSM (B <- L^-1 B).  trsm_rec splits L at split_point(n), a multiple of 128, solves the top, updates the bottom with
one GEMM (k = n1, beta = 1) and recurses; a leaf (n <= 128) multiplies by the cached inverse X_i of its diagonal block.
With a forward error the leaves are not componentwise backward stable, so the bar is on the residual r = b - L x.
Leaf i: x_i = fl(X_i b~_i) = (X_i + E) b~_i with |E| <= gamma_nb |X_i|, hence
    b~_i - L_ii x_i = (I - L_ii X_i) b~_i - L_ii E b~_i,   |b~_i| <= |L_ii| |x_i| + |r_i|,
so |r_i| <= (eta_i + gamma_nb kappa_i) max_{rows of block i} (|L| |x|) (|L_ii| |x_i| <= |L| |x| on those rows, and
|r_i| in |b~_i| is of second order), where eta_i = || I - L_ii X_i ||_inf is the leaf inverse's own residual and
kappa_i = || |L_ii| |X_i| ||_inf the block condition number.  An update
b2 - L21 x1 adds at most gamma_{n1+2} (|L21| |x1| + |b2|) <= 2 gamma_{n1+2} (|L| |x|) to its rows; the n1 of the
levels above one row sum to at most n, so with d the recursion depth
    |b - L x|_r <= [eta_i + gamma_128 kappa_i + 2 gamma_{n + 2 d}] max_{rows s of r's block} (|L| |x|)_s.
(trans = 1 is the same statement for L^T, with L_ii^T, X_i^T.)  eta_i is computed from the device's X_i: the leaf
inverses come from the factorisation, which has its own tests; this bar isolates the solve.  For kappa_i up to 1e6
the kappa term dominates, so the ill-conditioned cases check it at its own size.

L^-1 (trtri_rec).  The recursion writes X21 = -X22 fl(L21 X11) with two GEMMs (k = n1 then k = n2), so the identity
it controls is local: for every split of the recursion, against the device's own X11 and X22,
    |X21 + X22 L21 X11| <= (gamma_{n1} + gamma_{n2} + gamma_{n1} gamma_{n2}) |X22| |L21| |X11|       elementwise,
and the diagonal blocks equal the cached inverses exactly (put_dinv_kernel copies them).  These identities determine
X up to roundings; a global residual |X L - I| adds only products of block condition numbers on top of them.

lauum (C = X^T X, lower).  Every lower entry is a sum of n products split over the recursion: the leaf GEMM and one
beta = 1 GEMM per level above, each adding two roundings, so |C_dev - X^T X| <= gamma_{n + 2 d} |X|^T |X|, measured
against the device's own X.

chol_adjoint (G = -sym(L^-T Phi(T) L^-1)).  Two solves with L^T: by the TRSM bar each has a normwise residual
||r||_F <= eps_s ||L||_2 ||x||_F with eps_s = sqrt(128 n) (gamma_128 kappa_max + eta_max + 2 gamma_{n+2d}) (the
block maximum of |L| |x| over 128 rows costs sqrt(128), |L| against L costs sqrt(n)); the forward error of each is
then at most kappa_2(L) eps_s ||x||.  ||Phi(T)||_F <= ||T||_F and each solve multiplies by at most ||L^-1||_2, so
    max |G_dev - G| <= ||G_dev - G||_F <= (2 kappa_2(L) eps_s + 2 u) ||L^-1||_2^2 ||T||_F,
and the fp64 LAPACK reference adds the same amount again (factor 2 in `chol_adjoint_bar`)."""
from __future__ import annotations

import numpy as np
import scipy.linalg as sla

U = 2.0 ** -53
U_LD = 2.0 ** -64
NB = 128
GEMM_LOWER_ONLY, GEMM_A_LOWER, GEMM_COLSUMSQ = 1, 2, 4
SKINNY_N = 16
TILES = [(128, 128), (128, 64), (128, 32), (64, 128), (32, 128)]


def gamma(k, u=U):
    k = np.asarray(k, dtype=np.float64)
    return k * u / (1.0 - k * u)


def split_point(n):
    """potrf.cu::split_point and grad.cu::split128 (the same rule)."""
    return ((n // NB + 1) // 2) * NB


def depth(n):
    d = 0
    while n > NB:
        n1 = split_point(n)
        n, d = max(n1, n - n1), d + 1
    return d


# ---- tile selection mirror -------------------------------------------------------------------------------------------
def dmma_tile(m, n, flags=0, alias=None, tb=0, k=0, dtype=np.float64):
    """The kernel gemm.cu::gemm_t launches for C[m, n]: "skinny", "tf32" (fp32 3xTF32 path) or the tile (BM, BN) of
    launch_dmma / launch_simt (the same rules).  alias: None, "A" (C == A) or "B" (C == B)."""
    if m <= 0 or n <= 0:
        return None
    if n <= SKINNY_N and not tb and flags == 0 and alias is None:
        return "skinny"
    if np.dtype(dtype) == np.float32 and k >= 64 and m >= 64 and n >= 64 and m * n * k >= 2.0e8:
        return "tf32"
    t128 = -(-m // 128) * -(-n // 128)
    if t128 >= 120 or flags & GEMM_COLSUMSQ:
        return (128, 128)
    if alias == "B" or (m <= 128 and alias != "A"):
        return (128, 64) if -(-n // 64) >= 100 else (128, 32)
    if alias == "A" or n <= 128:
        return (64, 128) if -(-m // 64) >= 100 else (32, 128)
    return (64, 128) if -(-m // 64) * -(-n // 128) >= 100 else (32, 128)


def tiles_written(m, n, tile, flags):
    """Boolean [m, n] mask of the entries the tiled kernel may store: every tile, except with LOWER_ONLY those whose
    first column lies right of their last row (gemm_dmma_kernel's early return)."""
    bm, bn = tile
    mask = np.ones((m, n), dtype=bool)
    if flags & GEMM_LOWER_ONLY:
        for m0 in range(0, m, bm):
            for n0 in range(0, n, bn):
                if n0 > m0 + bm - 1:
                    mask[m0:m0 + bm, n0:n0 + bn] = False
    return mask


def edge_indices(n, rng, extra=24, step=32):
    """Every tile-edge index (multiples of 32 and the ones before them), the last index and `extra` random ones."""
    idx = set()
    for e in range(0, n + 1, step):
        idx.update(i for i in (e - 1, e) if 0 <= i < n)
    idx.add(n - 1)
    if n > 0:
        idx.update(rng.integers(0, n, size=min(extra, n)).tolist())
    return np.array(sorted(idx), dtype=np.int64)


# ---- GEMM ------------------------------------------------------------------------------------------------------------
def opmat(M, t):
    return M.T if t else M


def gemm_ref(A, B, C0, alpha, beta, ta, tb, rows, cols, a_lower=False):
    """Long double alpha op(A)[rows] op(B)[:, cols] + beta C0[rows][:, cols] and its bar."""
    As = np.tril(A) if a_lower else A
    oa, ob = opmat(As, ta)[rows], opmat(B, tb)[:, cols]
    k = oa.shape[1]
    prod = oa.astype(np.longdouble) @ ob.astype(np.longdouble)
    mag = np.abs(alpha) * (np.abs(oa) @ np.abs(ob))
    ref = np.longdouble(alpha) * prod
    if beta != 0.0:
        c0 = C0[rows][:, cols]
        ref = ref + np.longdouble(beta) * c0.astype(np.longdouble)
        mag = mag + abs(beta) * np.abs(c0)
    bar = (gamma(k + 2) + (k + 2) * U_LD) * mag * (1 + 4 * U) + np.finfo(np.float64).tiny
    return ref, bar


def ratio(err, bar):
    """max err / bar (0 for an exact result); inf when any error is not finite (a NaN never passes)."""
    q = np.asarray(err, dtype=np.float64) / bar
    if not np.isfinite(q).all():
        return float("inf")
    return float(np.max(q)) if q.size else 0.0


# ---- TRSM ------------------------------------------------------------------------------------------------------------
def block_stats(L, Xblocks, trans):
    """(kappa_i, eta_i) per 128-block: kappa_i = || |Lt_ii| |Xt_i| ||_inf and eta_i = || I - Lt_ii Xt_i ||_inf
    with Lt = L (trans = 0) or L^T, Xt_i the device's inverse of the block (transposed with L), taken whole: the leaf
    GEMM reads the full 128 x 128 block."""
    n = L.shape[0]
    kap, eta = [], []
    for b, X in enumerate(Xblocks):
        o = b * NB
        nb = min(NB, n - o)
        Lii = np.tril(L[o:o + nb, o:o + nb])
        Xi = X[:nb, :nb]
        if trans:
            Lii, Xi = Lii.T, Xi.T
        kap.append(np.abs(Lii) @ np.abs(Xi))
        R = np.eye(nb, dtype=np.longdouble) - Lii.astype(np.longdouble) @ Xi.astype(np.longdouble)
        eta.append(float(np.max(np.abs(R).astype(np.float64).sum(axis=1))))
        kap[-1] = float(np.max(kap[-1].sum(axis=1)))
    return np.array(kap), np.array(eta)


def trsm_check(L, B0, X, Xblocks, trans, cols, u=U):
    """(ratio, kappa_max, eta_max) of the residual |b - Lt x| for the sampled right-hand sides `cols` against the TRSM
    bar, with unit roundoff u for the arithmetic of the solve (2^-53 for fp64)."""
    n = L.shape[0]
    Lt = np.tril(L).T if trans else np.tril(L)
    kap, eta = block_stats(L, Xblocks, trans)
    x = X[:, cols]
    r = B0[:, cols].astype(np.longdouble) - Lt.astype(np.longdouble) @ x.astype(np.longdouble)
    mag = np.abs(Lt) @ np.abs(x)
    nblk = -(-n // NB)
    bar = np.empty_like(mag)
    for b in range(nblk):
        o = b * NB
        nb = min(NB, n - o)
        c = eta[b] + gamma(min(n, NB), u) * kap[b] + 2 * gamma(n + 2 * depth(n), u) + n * U_LD
        bar[o:o + nb] = c * mag[o:o + nb].max(axis=0, keepdims=True)
    bar = bar * (1 + 4 * u) + np.finfo(np.float64).tiny
    return ratio(np.abs(r), bar), kap.max(), eta.max()


# ---- inverse chain ---------------------------------------------------------------------------------------------------
def splits(n, o=0):
    """Every split (offset, n1, n2) of the trtri / lauum recursion over n, top first."""
    if n <= NB:
        return []
    n1 = split_point(n)
    return [(o, n1, n - n1)] + splits(n1, o) + splits(n - n1, o + n1)


def trtri_check(L, X, rng, ncols=40):
    """Worst ratio of |X21 + X22 L21 X11| to its bar over every split (sampled columns of X21, every row)."""
    worst = 0.0
    for o, n1, n2 in splits(L.shape[0]):
        X11 = np.tril(X[o:o + n1, o:o + n1])
        X22 = np.tril(X[o + n1:o + n1 + n2, o + n1:o + n1 + n2])
        L21 = L[o + n1:o + n1 + n2, o:o + n1]
        X21 = X[o + n1:o + n1 + n2, o:o + n1]
        cols = edge_indices(n1, rng, extra=ncols // 2)
        T = L21.astype(np.longdouble) @ X11[:, cols].astype(np.longdouble)
        ident = X21[:, cols].astype(np.longdouble) + X22.astype(np.longdouble) @ T
        mag = np.abs(X22) @ (np.abs(L21) @ np.abs(X11[:, cols]))
        bar = (gamma(n1) + gamma(n2) + gamma(n1) * gamma(n2) + (n1 + n2) * U_LD) * mag * (1 + 4 * U)
        worst = max(worst, ratio(np.abs(ident), bar + np.finfo(np.float64).tiny))
    return worst


def lauum_check(X, rows, cols):
    """Ratio of |C - X^T X| on the sampled lower entries (rows x cols, i >= j) to gamma_{n+2d} |X|^T |X|; returns a
    function of the device's C."""
    n = X.shape[0]
    Xl = np.tril(X)
    ref = Xl[:, rows].T.astype(np.longdouble) @ Xl[:, cols].astype(np.longdouble)
    mag = np.abs(Xl[:, rows]).T @ np.abs(Xl[:, cols])
    bar = (gamma(n + 2 * depth(n)) + n * U_LD) * mag * (1 + 4 * U) + np.finfo(np.float64).tiny
    low = rows[:, None] >= cols[None, :]

    def check(C):
        err = np.abs(C[np.ix_(rows, cols)].astype(np.longdouble) - ref).astype(np.float64)
        return ratio(err[low], bar[low])

    return check


def chol_adjoint_ref(L, T):
    """fp64 LAPACK G = -sym(L^-T Phi(T) L^-1)."""
    Phi = np.tril(T, -1) + 0.5 * np.diag(np.diag(T))
    Li = sla.solve_triangular(L, np.eye(L.shape[0]), lower=True)
    Z = Li.T @ Phi @ Li
    return -0.5 * (Z + Z.T)


def chol_adjoint_bar(L, T, kap_max, eta_max):
    n = L.shape[0]
    s = np.linalg.svd(np.tril(L), compute_uv=False)
    eps_s = np.sqrt(NB * n) * (gamma(min(n, NB)) * kap_max + eta_max + 2 * gamma(n + 2 * depth(n)))
    return 2 * (2 * (s[0] / s[-1]) * eps_s + 2 * U) * np.linalg.norm(T) / s[-1] ** 2


# ---- test matrices ---------------------------------------------------------------------------------------------------
def block_kappa(L):
    """max_i || |L_ii| |L_ii^-1| ||_inf over the 128-diagonal blocks."""
    k = 0.0
    for o in range(0, L.shape[0], NB):
        Lii = np.tril(L[o:o + NB, o:o + NB])
        Xi = sla.solve_triangular(Lii, np.eye(Lii.shape[0]), lower=True)
        k = max(k, float(np.max((np.abs(Lii) @ np.abs(Xi)).sum(axis=1))))
    return k


def factor_with_block_cond(n, rng, cond=1.0):
    """Lower factor with positive diagonal whose 128-diagonal blocks have condition numbers kappa_i up to about
    `cond`: the blocks are I + s N (N strictly lower, standard normal), whose inverses grow with s; s is found by
    bisection.  The blocks below the diagonal are N(0, 1/4n)."""
    L = np.tril(rng.standard_normal((n, n)), -1) * (0.5 / np.sqrt(n))
    N = np.tril(rng.standard_normal((n, n)), -1)
    blk = np.zeros((n, n), dtype=bool)
    for o in range(0, n, NB):
        blk[o:o + NB, o:o + NB] = True

    def make(s):
        return np.where(blk, s * N, L) + np.eye(n)

    if cond <= 1.0:
        return make(0.1 / np.sqrt(NB))
    lo, hi = 0.0, 1.0
    while block_kappa(make(hi)) < cond:
        hi *= 2
    for _ in range(16):
        mid = 0.5 * (lo + hi)
        lo, hi = (mid, hi) if block_kappa(make(mid)) < cond else (lo, mid)
    return make(hi)


# ---- CPU emulations of the recursions (fp64 NumPy, same splits, inverse-based leaves) ---------------------------------
def leaf_inverses(L):
    n = L.shape[0]
    out = []
    for o in range(0, n, NB):
        nb = min(NB, n - o)
        out.append(sla.solve_triangular(np.tril(L[o:o + nb, o:o + nb]), np.eye(nb), lower=True))
    return out


def emu_trsm(trans, L, B, Xb, o=0):
    n = L.shape[0]
    if n <= NB:
        X = Xb[o // NB][:n, :n]
        return (X.T if trans else X) @ B
    n1 = split_point(n)
    L21 = L[n1:, :n1]
    B = B.copy()
    if not trans:
        B[:n1] = emu_trsm(0, L[:n1, :n1], B[:n1], Xb, o)
        B[n1:] = emu_trsm(0, L[n1:, n1:], B[n1:] - L21 @ B[:n1], Xb, o + n1)
        return B
    B[n1:] = emu_trsm(1, L[n1:, n1:], B[n1:], Xb, o + n1)
    B[:n1] = emu_trsm(1, L[:n1, :n1], B[:n1] - L21.T @ B[n1:], Xb, o)
    return B


def emu_trtri(L, Xb):
    """L^-1 as grad.cu::potri_lower's put_dinv + trtri_rec computes it."""
    n = L.shape[0]
    X = np.tril(L).copy()
    for b, Xi in enumerate(Xb):
        o = b * NB
        nb = Xi.shape[0]
        X[o:o + nb, o:o + nb] = np.tril(Xi)

    def rec(o, n):
        if n <= NB:
            return
        n1 = split_point(n)
        rec(o, n1)
        rec(o + n1, n - n1)
        X11 = np.tril(X[o:o + n1, o:o + n1])
        X22 = np.tril(X[o + n1:o + n, o + n1:o + n])
        Tt = X11.T @ X[o + n1:o + n, o:o + n1].T
        X[o + n1:o + n, o:o + n1] = -(X22 @ Tt.T)

    rec(0, n)
    return X


def emu_lauum(X):
    n = X.shape[0]
    C = np.zeros((n, n))

    def rec(o, n):
        A = X[o:o + n, o:o + n]
        if n <= NB:
            C[o:o + n, o:o + n] = np.tril(A).T @ np.tril(A)
            return
        n1 = split_point(n)
        rec(o, n1)
        rec(o + n1, n - n1)
        A21, A22 = A[n1:, :n1], np.tril(A[n1:, n1:])
        C[o:o + n1, o:o + n1] += A21.T @ A21
        C[o + n1:o + n, o:o + n1] = A22.T @ A21

    rec(0, n)
    return C
