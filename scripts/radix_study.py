"""Round-2 study (CPU, NumPy): digit radix of the int8 tensor-core trailing updates.  Radix 128 (round 1: digits in [-64, 64], S
planes resolve 2^-(7S - 1) of the static row scale) against radix 256 (balanced base-256 digits in [-128, 127], top digit
in [-65, 65]: S planes resolve 2^-(8S - 2)), S(S+1)/2 int8 MMAs per k-step either way.  Emulates the recursive
factorisation of potrf.cu with static row exponents for K >= 256 and reports the error of L and of sum log diag L against
LAPACK for a range of noise levels (conditioning ~ (1 + noise) / noise); pick_slices() in potrf.cu is set from this table.

    python scripts/radix_study.py [N] [hard]
"""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from oracle import gp_oracle as O

NB = 128


def digits(P, e, S, bits):
    v = P * np.exp2(6.0 - e)[:, None]
    if bits == 7:
        D = np.empty((S,) + P.shape, dtype=np.int64)
        for s in range(S):
            d = np.clip(np.rint(v), -64, 64)
            v = (v - d) * 128.0
            D[s] = d
        return D
    I = np.rint(v * 2.0 ** (8 * (S - 1))).astype(np.int64)   # |v| < 64: |I| < 2^54 for S = 7, 2^62 for S = 8
    D = np.empty((S,) + P.shape, dtype=np.int64)
    for s in range(S - 1, 0, -1):
        d = ((I + 128) & 255) - 128
        D[s] = d
        I = (I - d) >> 8
    D[0] = I
    assert np.abs(D[0]).max() <= 65 and D.min() >= -128 and D.max() <= 127
    return D


SQUARE_TERM = False   # even S: also keep the (S/2, S/2) digit product -- the only dropped order-S term with a non-zero mean
                      # on the diagonal of C (d^2 > 0), i.e. the systematic part of the error of sum log diag L


def sliced_update(C, P, n, e_rows, S, bits):
    m = P.shape[0]
    D = digits(P, e_rows, S, bits)
    rs = np.exp2(e_rows - 6.0)
    acc = np.zeros((m, n))
    for g in range(S):
        a = np.zeros((m, n), dtype=np.int64)
        for s in range(g + 1):
            a += D[s] @ D[g - s][:n].T
        assert np.abs(a).max() < 2 ** 31
        acc += a * 2.0 ** (-bits * g)
    if SQUARE_TERM and S % 2 == 0:
        acc += (D[S // 2] @ D[S // 2][:n].T) * 2.0 ** (-bits * S)
    C -= acc * rs[:, None] * rs[None, :n]


def potrf_rec(A, n, e_static, S, bits, off=0):
    rows = A.shape[0]
    if n <= NB:
        A[:n, :n] = np.linalg.cholesky(A[:n, :n])
        if rows > n:
            A[n:, :n] = np.linalg.solve(A[:n, :n], A[n:, :n].T).T
        return
    n1 = ((n // NB + 1) // 2) * NB
    potrf_rec(A, n1, e_static, S, bits, off)
    P = A[n1:, :n1]
    C = A[n1:, n1:n]
    if n1 >= 256 and S:
        sliced_update(C, P, n - n1, e_static[off + n1:off + rows], S, bits)
    else:
        C -= P @ P[:n - n1].T
    potrf_rec(A[n1:, n1:], n - n1, e_static, S, bits, off + n1)


def run(N, noise, S, bits, hard=False):
    d = O.make_data(2, N, 8, 1)
    if hard:   # numerically low-rank: smooth kernel on 1-D inputs, lambda_min = noise, lambda_max ~ N
        x = np.sort(np.random.default_rng(3).uniform(0, 1, (N, 1)), axis=0)
        K = O.SquaredExponential(lengthscales=0.5)(x) + noise * np.eye(N)
    else:
        K = O.Matern52(lengthscales=np.sqrt(8.0))(d["X"]) + noise * np.eye(N)
    Lx = np.linalg.cholesky(K)
    A = K.copy()
    e = np.floor(np.log2(np.sqrt(np.diag(K)))) + 1.0
    try:
        potrf_rec(A, N, e, S, bits)
    except np.linalg.LinAlgError:
        return float("nan"), float("nan"), float("nan")
    L = np.tril(A)
    y = d["Y"][:, 0]
    quad = lambda LL: float(np.sum(np.linalg.solve(LL, y) ** 2))
    lml = lambda LL: -0.5 * quad(LL) - np.sum(np.log(np.diag(LL)))
    return (np.abs(L - Lx).max() / np.abs(Lx).max(), abs(np.sum(np.log(np.diag(L))) - np.sum(np.log(np.diag(Lx)))),
            abs(lml(L) - lml(Lx)) / abs(lml(Lx)))


if __name__ == "__main__":
    N = int(sys.argv[1]) if len(sys.argv) > 1 else 1024
    hard = len(sys.argv) > 2 and sys.argv[2] == "hard"
    print(f"N = {N}; columns: max|dL|/max|L|, |d sum log diag L|, relative LML error")
    for noise in (1e-1, 1e-2, 1e-3, 1e-4, 1e-5, 1e-6, 1e-7, 1e-8):
        row = [f"noise {noise:.0e} (cond ~ {(1 + noise) / noise:.1e})"]
        for bits, S, sq in ((0, 0, 0), (7, 7, 0), (7, 8, 0), (8, 6, 0), (8, 6, 1), (8, 7, 0), (8, 8, 0)):
            SQUARE_TERM = bool(sq)
            eL, dl, rl = run(N, noise, S, bits, hard)
            row.append(f"{'fp64' if not S else f'r{1 << bits} S={S}' + ('+sq' if sq else '')}: {eL:.1e} {dl:.1e} {rl:.1e}")
        print(" | ".join(row))
