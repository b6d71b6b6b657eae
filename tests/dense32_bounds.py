"""Error bars, a CPU model of the arithmetic and mirrors of the dispatch for the fp32 dense products of the SGPR and
SVGP objectives, CPU only.

The kernels are gemm_tf32.cu (3xTF32 on warpgroup MMAs, its split-K and its batched column sums of squares) and the
fp32 CUDA-core kernels of gemm.cu (the tiled SIMT GEMM and the skinny kernel, n <= 16).

Model of the 3xTF32 kernel (`emulate_tf32`).  The pre-pass splits every operand a = hi + lo with hi = rna_tf32(a),
lo = rna_tf32(a - hi); every k8 step issues three MMAs, lo*hi, hi*lo and hi*hi, in that order, into one accumulator d.
The MMA is modelled pessimistically (no guard bits): the eight TF32 products are exact, each of the nine addends
(d and the products) is truncated to 24 bits at the exponent of the largest, the exact sum of those is truncated to
fp32.  d starts from zero every TF_KP = 64 k and is then added round-to-nearest into an fp32 register accumulator.
The mutants the tests must catch are modelled the same way: "2x" drops the hi*lo MMA, "1x" keeps hi*hi only, and
run=None promotes once per K range.

Worst-case bars, per element, unit roundoff u (2^-24 for fp32) a parameter:
  3xTF32: the split loses at most 2^-20 |a||b| per product (hi*hi + hi*lo + lo*hi misses lo*lo and the rounding of
    lo; test_tf32_split_model checks it).  One MMA loses at most 9 ulps of its largest addend, at most
    U_MMA = 9 * 2^-23 of the magnitude |d| + sum |p| it adds up, and a run of 24 MMAs at most 24 U_MMA of the
    magnitude of its 64 products; the runs' errors add up to 24 U_MMA sum_k |a_k||b_k|.  The promotions are an fp32
    sum of ceil(K / 64) runs (gamma_runs), alpha * acc and beta * C0 + x one rounding each, and split-K adds the
    prescaling of C and nsplit atomic additions:
        |C_dev - C| <= (2^-20 + 24 U_MMA + gamma_{runs + nsplit + 2}(u)) (|alpha| |op(A)||op(B)| + |beta| |C0|).
  CUDA-core GEMM and skinny kernel: any order of fp32 fmas, gamma_{k+2}(u) of the same magnitude
    (dense64_bounds.gemm_ref with u = 2^-24).
  COLSUMSQ: with y = alpha op(A) op(B) and |y^ - y| <= g s (s = |alpha| |op(A)||op(B)|, g the GEMM bar above),
    |sum y^2 - sum y^2| <= sum (2 |y| g s + g^2 s^2); the epilogue adds two rows per thread with fmaf and three xor
    shuffles (5 roundings per 16-row warp slice), then one fp32 atomicAdd per slice onto the prefilled value v0:
    gamma_{5 + m/16 + 1}(u) (|v0| + sum (|y| + g s)^2).  In the SVGP forward v0 = fvar0 = Kdiag - sum A^2 comes
    from colsumsq_kernel (fp64 sums, one fp32 atomicAdd per 8 x 32 block): its own error is a bar of its own.

The worst-case bars hold for any correctly working kernel, so they are loose (a typical ratio is 1e-3): a kernel that
lost one of its correction MMAs stays inside them.  Two statistics see what they cannot:
  rms_rel: the RMS over many entries of (C_dev - C) / (|alpha| |op(A)||op(B)| + |beta| |C0|).  A lost 2^-12 correction
    term gives about 2^-12 * 1.3 / sqrt(K) on N(0,1) data; RMS_C / sqrt(K) with RMS_C = 2^-16 sits a decade below that
    and a decade above the model's correct kernel at K = 2048 and K = 1e5 (test_dense32_bounds).
  mean signed relative error over the diagonal of A A^T: every product is positive, so the truncation cannot cancel.
    BIAS_BAR = 3e-6: the model's correct kernel is at -7e-7 / -9e-7 (K = 2048 / 1e5), promoting once per K range at
    -3.5e-5 / -2e-3."""
from __future__ import annotations

import numpy as np

from tests import dense64_bounds as DB

U32 = 2.0 ** -24
U_SPLIT = 2.0 ** -20
U_MMA = 9 * 2.0 ** -23
TF_BM = TF_BN = 128
TF_KS, TF_KP = 16, 64
MMAS_PER_RUN = 3 * TF_KP // 8
RMS_C = 2.0 ** -16
BIAS_BAR = 3e-6
SKINNY_N = 16
GEMM_LOWER_ONLY, GEMM_A_LOWER, GEMM_COLSUMSQ = DB.GEMM_LOWER_ONLY, DB.GEMM_A_LOWER, DB.GEMM_COLSUMSQ
SMS = 132


# ---- model -----------------------------------------------------------------------------------------------------------
def rna_tf32(x: np.ndarray) -> np.ndarray:
    """cvt.rna.tf32.f32: round the fp32 mantissa to 10 bits, ties away from zero."""
    u = x.astype(np.float32).view(np.uint32).astype(np.uint64)
    u = ((u + 0x1000) & 0xFFFFE000).astype(np.uint32)
    return u.view(np.float32)


def split(x):
    hi = rna_tf32(x)
    lo = rna_tf32((x.astype(np.float32) - hi).astype(np.float32))
    return hi, lo


def _rz(x, bits=24):
    """x rounded toward zero to `bits` significant bits."""
    m, e = np.frexp(x)
    return np.ldexp(np.trunc(np.ldexp(m, bits)), e - bits)


def mma(d, p):
    """One MMA step of the model: d + sum of the exact products p[..., 8], addends truncated at the largest exponent,
    the sum truncated to fp32."""
    t = np.concatenate([d[..., None], p], axis=-1)
    _, e = np.frexp(np.abs(t).max(axis=-1))
    q = np.ldexp(1.0, e - 24)[..., None]
    return _rz((np.trunc(t / q) * q).sum(axis=-1))


def emulate_tf32(a, b, mode="3x", run=TF_KP):
    """fp32 op(A) op(B) as the model of gemm_tf32_kernel computes it (alpha = 1, beta = 0, one k split): a [..., K] rows
    of op(A) and b [..., K] columns of op(B), broadcast against each other.  mode "3x" (the kernel), "2x" (no hi*lo
    MMA), "1x" (hi*hi only); run = None promotes once per K range."""
    ah, al = (x.astype(np.float64) for x in split(a))
    bh, bl = (x.astype(np.float64) for x in split(b))
    K = a.shape[-1]
    terms = {"3x": [(al, bh), (ah, bl), (ah, bh)], "2x": [(al, bh), (ah, bh)], "1x": [(ah, bh)]}[mode]
    shape = np.broadcast_shapes(a.shape[:-1], b.shape[:-1])
    acc = np.zeros(shape, np.float32)
    run = run or K
    for r0 in range(0, K, run):
        d = np.zeros(shape)
        for k in range(r0, min(r0 + run, K), 8):
            for x, y in terms:
                d = mma(d, x[..., k:k + 8] * y[..., k:k + 8])
        acc = (acc + d.astype(np.float32)).astype(np.float32)
    return acc


def emulate_colsumsq(Y, v0):
    """gemm_tf32_kernel's COLSUMSQ epilogue on the fp32 products Y [m, n] (alpha folded in), onto v0 [n]: per 16-row
    warp slice, thread (g, c) takes rows g and g + 8 with fmaf, three xor shuffles add the 8 threads of a column, one
    fp32 atomicAdd per slice (here in slice order)."""
    Y = np.asarray(Y, np.float32)
    m, n = Y.shape
    Yp = np.zeros((-(-m // 16) * 16, n), np.float32)
    Yp[:m] = Y
    out = np.asarray(v0, np.float32).copy()
    for r in range(0, Yp.shape[0], 16):
        x0, x1 = Yp[r:r + 8].astype(np.float64), Yp[r + 8:r + 16].astype(np.float64)
        s = (x0 * x0).astype(np.float32)
        s = (x1 * x1 + s).astype(np.float32)                   # fmaf: one rounding
        for mask in (1, 2, 4):                                 # lanes xor 4, 8, 16 = row groups xor 1, 2, 4
            s = (s + s[np.arange(8) ^ mask]).astype(np.float32)
        out = (out + s[0]).astype(np.float32)
    return out


# ---- bars ------------------------------------------------------------------------------------------------------------
def gamma(k, u=U32):
    return DB.gamma(k, u)


def g_tf32(k, nsplit=1, u=U32):
    """Relative per-element bar of the 3xTF32 GEMM (see the module docstring)."""
    runs = -(-k // TF_KP) + 1
    return U_SPLIT + MMAS_PER_RUN * U_MMA * (1 + 2.0 ** -9) + gamma(runs + nsplit + 2, u)


def g_simt(k, u=U32):
    return gamma(k + 2, u)


def g_ref(k):
    """Error of the fp64 reference products the tests compare with."""
    return DB.gamma(k + 2)


def colsumsq_bar(y, s, g, m, v0):
    """Bar on |sum_i y^_i^2 + v0 - (sum_i y_i^2 + v0)| for one batch: y [m, n] exact products, s [m, n] their
    magnitudes, g the GEMM's relative bar."""
    v0 = np.broadcast_to(np.abs(np.asarray(v0, np.float64)), y.shape[1:])
    ay = np.abs(y)
    prod = (2 * ay * g * s + (g * s) ** 2).sum(axis=0)
    return prod + gamma(5 + -(-m // 16) + 1) * (v0 + ((ay + g * s) ** 2).sum(axis=0))


def rms_bar(k):
    return RMS_C / np.sqrt(k)


def rms_rel(err, mag):
    e = np.asarray(err, np.float64) / mag
    return float(np.sqrt(np.mean(e ** 2))) if np.isfinite(e).all() else float("inf")


def signed_bias(diag_dev, diag_ref):
    return float(np.mean((np.asarray(diag_dev, np.float64) - diag_ref) / diag_ref))


# ---- dispatch mirrors ------------------------------------------------------------------------------------------------
def gemm_kernel(m, n, k, flags=0, alias=None, tb=0, engine="tf32"):
    """What gemm.cu::gemm_t runs for an fp32 C[m, n]: "skinny", "tf32" or "simt" (engine = "simt":
    GPK_FP32_ENGINE=simt)."""
    if m <= 0 or n <= 0:
        return None
    if n <= SKINNY_N and not tb and flags == 0 and alias is None:
        return "skinny"
    if engine == "tf32" and k >= 64 and m >= 64 and n >= 64 and m * n * k >= 2.0e8:
        return "tf32"
    return "simt"


def tf32_launch(m, n, k, flags=0, batch=1, cluster=2, sms=SMS):
    """(cl, nsplit) of gemm_tf32: cl = 2 row tiles per cluster unless there is one row tile (or GPK_TF32_CLUSTER=1),
    K split while the work units cannot fill the SMs and every split keeps >= 64 stages; never with COLSUMSQ."""
    mt = m * batch
    ntm, ntn = -(-mt // TF_BM), -(-n // TF_BN)
    KB = -(-k // TF_KS)
    cl = cluster if ntm >= 2 else 1
    lower = bool(flags & GEMM_LOWER_ONLY)
    nunits = sum(1 for tn in range(ntn) for t0 in range(0, ntm, cl)
                 if not (lower and tn * TF_BN > (t0 + cl - 1) * TF_BM + TF_BM - 1))
    nsplit = 1
    while nunits * cl * nsplit < sms and KB // (nsplit * 2) >= 64 and nsplit < 64:
        nsplit *= 2
    if flags & GEMM_COLSUMSQ:
        nsplit = 1
    return cl, nsplit


def svgp_fvar_path(B, M, Pl, q_diag, dtype=np.float32, batched_env=True, engine="tf32"):
    """Which kernel fused.cu::svgp_forward runs for fvar: "q_diag" (colsumsq_kernel with row weights), "batched"
    (one gemm_tf32 launch over the Pl latents), or per latent the kernel gemm_t picks for the COLSUMSQ product."""
    if q_diag:
        return "q_diag"
    tf = gemm_kernel(M, B, M, GEMM_A_LOWER | GEMM_COLSUMSQ, engine=engine) == "tf32"
    if batched_env and np.dtype(dtype) == np.float32 and Pl > 1 and M % 256 == 0 and tf:
        return "batched"
    return "tf32" if tf and np.dtype(dtype) == np.float32 else "simt"


def edge_indices(n, rng, extra=24, step=32):
    return DB.edge_indices(n, rng, extra, step)
