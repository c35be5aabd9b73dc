"""fp64 attention reference, its error bound, and adversarial input generators for the attention tests.

Reference.  O64 = softmax(S) V, S = scale * Q K^T, computed directly (not online) in float64 from the fp16 inputs, with
lse64 = logsumexp(S), the sensitivity sigma[i, d] = sum_j p_ij |v_jd|, tau[i, d] = sum_j |v_jd| / l_i
(l_i = sum_j exp(S_ij - max_j S_ij)) and rho[i], a bound in nats on the fp32 error of any score of row i.
`reference` takes numpy arrays (CPU self-check) or torch tensors (GPU tests, computed on the device).

Bound (`o_bound`).  What the kernel (csrc/attn_sm90.cuh, softmax_math.cuh, DESIGN.md §5) does to O, term by term:

  * P is rounded to fp16 before P V, the row sum l is taken from the unrounded fp32 values: every term of the
    numerator moves by at most u = 2^-11 relative, i.e. O by at most u * sigma (c = 1 below).  A P below the
    fp16 normal range (2^-14) is rounded on the fixed 2^-25 grid instead: at most 2^-25 sum_j |v_j| / l = 2^-25 tau.
  * Every weight p_j carries a relative error e_j that enters numerator and l alike, which moves O by at most
    max|e| * sum_j p_j |v_j - O| <= max|e| (sigma + |O|).  Its parts: the FMA-pipe polynomial on a quarter of the
    keys at D <= 128 (7.6e-5, softmax_math.cuh), ex2.approx (2^-21 taken, for the key and for the rescale factor
    alpha), the fp32 rounding of x = s * scale * log2e - m and of scale * log2e (2^-20 covers |x| <= 126), and
    the error of the fp32 score itself, 2 rho (e^rho - 1 <= 2 rho for rho < 1).  rho assumes each k16 wgmma step
    adds its 16 exact fp16 products with an error of at most 16 * 2^-23 of their magnitude and every accumulator
    add rounds once: rho_i = scale * (ceil(D/16) + 16) * 2^-23 * max_j sum_d |q_id k_jd|.  Inputs whose scores are
    exact in fp32 (integer multiples of one fp16 value, `one_hot`) pass exact_scores=True and get rho = 0.
  * fp32 sums: l is summed in fp32 (N/4 keys per thread, two shuffles, one multiply-add per key block):
    (N/4 + 2 ceil(N/64) + 4) 2^-23 relative, moving O by that times |O|; P V accumulates in fp32 on the tensor cores
    (ceil(N/16) + 16 + ceil(N/64)) 2^-23 of sigma by the same model as rho.
  * O is rounded once to fp16: 2^-11 |O| (relative), or 2^-25 absolute below the normal range (+ 2^-24 covers it).

  |O - O64| <= (u + acc) sigma + e (sigma + |O64|) + l_sum |O64| + 2^-25 tau  +  u |O64| + 2^-24

In the form c u sigma + u |O64| + 2^-24 this is c = 1 plus terms that stay below 0.2 u at default scale and
N <= 4096.  Nothing here is fitted to measurements.

lse (`lse_bound`).  lse = (m + log2 l) ln 2: l's relative error (poly, ex2, fp32 sum) moves it by as much, the scores by
rho, lg2.approx by <= 2^-20 ln 2, the roundings of m, of the sum and of the ln 2 product by <= 8 ulp = 2^-21 |lse|.

Fused RMS norm (`rms_reference`).  y = O r, r = g / sqrt(mean_d O^2 + 1e-5), evaluated on the fp32 O before its only
rounding: |dy| <= r b + |y| (mean_d(|O| b) / (mean_d O^2 + 1e-5) + (D + 4) 2^-24 + 2^-21) + u |y| + 2^-24, b the
bound of O without its rounding term (first order in b; rsqrt.approx taken as 2^-21).
"""
from __future__ import annotations

import math

import numpy as np
import torch

U16 = 2.0 ** -11                 # unit roundoff of fp16
EPS_POLY = 7.6e-5                # exp2_fma_pipe, max relative error (softmax_math.cuh)
EPS_EX2 = 2.0 ** -21             # ex2.approx.ftz.f32
EPS_X = 2.0 ** -20               # fp32 rounding of x = s * scale * log2e - m and of scale * log2e, |x| <= 126
LOG2E = 1.4426950408889634


def family(D, rms=False):
    """The kernel family fmha_dispatch picks for head dim D: (name, keys per block)."""
    if rms and D in (384, 512):
        return "rms-cluster", 64
    if D <= 64:
        return "D<=64", 128
    if D <= 128:
        return "64<D<=128", 64
    return "D>128", 64


def kernel_scale(D, scale=None):
    """The fp32 softmax scale the kernel uses: `scale`, or 1/sqrtf(D) when none is given."""
    if scale:
        return float(np.float32(scale))
    return float(np.float32(1.0) / np.sqrt(np.float32(D)))


# ------------------------------------------------------------------ reference
def _is_torch(x):
    return isinstance(x, torch.Tensor)


def _amax(x):
    return x.amax(dim=-1, keepdim=True) if _is_torch(x) else x.max(axis=-1, keepdims=True)


def _sum(x, axis=-1):
    return x.sum(dim=axis, keepdim=True) if _is_torch(x) else x.sum(axis=axis, keepdims=True)


def _f64(x):
    return x.double() if _is_torch(x) else np.asarray(x, dtype=np.float64)


def reference(q, k, v, scale, exact_scores=False):
    """Direct fp64 softmax attention of [..., N, D] inputs (numpy or torch) and the quantities the bound needs."""
    xp = torch if _is_torch(q) else np
    q, k, v = _f64(q), _f64(k), _f64(v)
    kt = k.swapaxes(-1, -2)
    s = (q @ kt) * scale
    mx = _amax(s)
    w = xp.exp(s - mx)
    l = _sum(w)
    p = w / l
    D = q.shape[-1]
    if exact_scores:
        rho = xp.zeros_like(mx)
    else:
        rho = scale * (math.ceil(D / 16) + 16) * 2.0 ** -23 * _amax(xp.abs(q) @ xp.abs(kt))
    return {"o": p @ v, "lse": (mx + xp.log(l))[..., 0], "sigma": p @ xp.abs(v),
            "tau": _sum(xp.abs(v), axis=-2) / l, "rho": rho, "N": k.shape[-2], "D": D}


def _weight_err(ref, poly):
    """Largest relative error of a softmax weight, per row."""
    return (EPS_POLY if poly else 0.0) + 2 * EPS_EX2 + EPS_X + 2 * ref["rho"]


def _lsum_err(N):
    return (N / 4 + 2 * math.ceil(N / 64) + 4) * 2.0 ** -23


def o_bound(ref, poly):
    """(bound before the fp16 rounding of O, bound of the fp16 O) per element; poly: D <= 128 kernels."""
    N = ref["N"]
    acc = (math.ceil(N / 16) + 16 + math.ceil(N / 64)) * 2.0 ** -23
    ao = abs(ref["o"])
    pre = ((U16 + acc) * ref["sigma"] + _weight_err(ref, poly) * (ref["sigma"] + ao) + _lsum_err(N) * ao
           + 2.0 ** -25 * ref["tau"])
    return pre, pre + U16 * ao + 2.0 ** -24


def lse_bound(ref, poly):
    e = (EPS_POLY if poly else 0.0) + 2 * EPS_EX2 + _lsum_err(ref["N"])
    return e + ref["rho"][..., 0] + 2.0 ** -20 * math.log(2.0) + 2.0 ** -21 * abs(ref["lse"])


def rms_reference(ref, g, pre):
    """y64 = rms_norm(O64) * g and its bound, from the reference and the pre-rounding bound `pre` of O."""
    xp = torch if _is_torch(ref["o"]) else np
    o = ref["o"]
    ms = _sum(o * o) / ref["D"] + 1e-5
    r = g / xp.sqrt(ms)
    y = o * r
    rel = _sum(abs(o) * pre) / ref["D"] / ms + (ref["D"] + 4) * 2.0 ** -24 + 2.0 ** -21
    return y, r * pre + abs(y) * rel + U16 * abs(y) + 2.0 ** -24


# ------------------------------------------------------------------ generators
GENERATORS = ("randn", "neg_scores", "front_max", "tail_max", "ramp_max", "one_hot")
# (generator, scale): None is the kernel's default 1/sqrt(D); 1.0 is sharp, 1e-3 near-uniform
VARIANTS = ([(g, None) for g in GENERATORS] + [(g, 1.0) for g in GENERATORS] + [("randn", 1e-3)])


def usable(gen, D):
    return gen != "one_hot" or D >= 32


def make_inputs(gen, B, H, N, D, kbn, scale=None, seed=0):
    """Seeded fp16 q, k, v [B, H, N, D] and, for `one_hot`, the permutation perm [B, H, N] with O[i] = V[perm[i]].

    randn       the baseline
    neg_scores  q = |randn| + 1, k = -(|randn| + 1): every real score is far below 0, so a zero-filled key past N
                (score 0, v = 0) would dominate its row
    front_max   the row maximum in key block 0, every later key >= 30 nats below (their exponentials reach the clamp)
    tail_max    the row maximum inside the last (ragged) key block, at the last key
    ramp_max    the maximum rises block by block: alpha << 1 at every block
    one_hot     k_j distinct +-1 codes, q_i = c k_perm(i) with a gap of >= 48 nats to every other key
    The three *_max generators put a bias t_j (nats) on coordinate 0: q[:, 0] = 1, k[j, 0] = t_j / scale; the other
    coordinates are randn, whose score noise has a standard deviation of about scale * sqrt(D) nats, and the gaps
    grow with it so that they hold at scale = 1 as well.  kbn: keys per block of the kernel under test.
    """
    rng = np.random.default_rng(seed)
    sc = kernel_scale(D, scale)
    shape = (B, H, N, D)

    def randn():
        return rng.standard_normal(shape, dtype=np.float32)

    perm = None
    if gen == "one_hot":
        assert D >= 32
        codes = np.where(rng.random(shape) < 0.5, -1.0, 1.0).astype(np.float32)
        # the codes of one head differ: their first bits spell the key index j
        nb = max(1, (N - 1).bit_length())
        codes[..., :nb] = np.where((np.arange(N)[:, None] >> np.arange(nb)) & 1, 1.0, -1.0)
        perm = rng.permuted(np.tile(np.arange(N), (B, H, 1)), axis=-1)
        c = np.float16(24.0 / sc)         # q.k_perm(i) - q.k_j >= 2 c: a gap of >= 48 nats
        k = codes
        q = np.take_along_axis(codes, perm[..., None], axis=2) * np.float32(c)
        v = randn()
        return (*(np.ascontiguousarray(x, dtype=np.float16) for x in (q, k, v)), perm)
    q, k, v = randn(), randn(), randn()
    if gen == "neg_scores":
        q, k = np.abs(q) + 1, -(np.abs(k) + 1)
    elif gen in ("front_max", "tail_max", "ramp_max"):
        noise = sc * math.sqrt(D)
        j = np.arange(N)
        blk = j // kbn
        if gen == "front_max":
            t = np.where(blk == 0, 0.0, -(30.0 + 8 * noise))
        elif gen == "tail_max":
            gap = 15.0 + 4 * noise
            t = np.where(blk == blk[-1], gap, 0.0)
            t[-1] += 4.0 + noise
        else:
            t = blk * (12.0 + 4 * noise)
        q[..., 0] = 1.0
        k[..., 0] = (t / sc)[None, None, :]
    elif gen != "randn":
        raise ValueError(gen)
    return q.astype(np.float16), k.astype(np.float16), v.astype(np.float16), perm


# ------------------------------------------------------------------ CPU restatements (self-check)
def exp2_fma_pipe(x):
    from test_softmax_math import exp2_fma_pipe as f
    return f(x)


def online(q, k, v, scale, kbn, kernel=False, poly_mask=0, skip_alpha_block=None, rms_g=0.0):
    """Online softmax over key blocks of kbn keys for one head ([N, D] numpy inputs).

    kernel=False: float64 throughout (equal to the direct reference up to float64 rounding); the mutations are
    applied to this form.  kernel=True restates the kernel's arithmetic: fp32 scores and statistics, x by one fused
    multiply-add, the keys `poly_mask` selects through exp2_fma_pipe, P rounded to fp16 before P V, fp32 O, the
    optional RMS norm on the fp32 row, one rounding to fp16.  Returns (O, lse)."""
    ft = np.float32 if kernel else np.float64
    c = ft(ft(scale) * ft(LOG2E))
    s_all = q.astype(ft) @ k.astype(ft).T
    n, nk = q.shape[0], k.shape[0]
    m = np.full((n, 1), -np.inf, ft)
    l = np.zeros((n, 1), ft)
    o = np.zeros((n, v.shape[1]), ft)
    with np.errstate(invalid="ignore", over="ignore"):
        for b0 in range(0, nk, kbn):
            s = s_all[:, b0:b0 + kbn]
            mn = np.maximum(m, (s.max(axis=1, keepdims=True) * c).astype(ft))
            alpha = np.exp2(m - mn).astype(ft)
            x = (s.astype(np.float64) * np.float64(c) - mn).astype(ft)
            p = np.exp2(x).astype(ft)
            if kernel and poly_mask:
                pair = (np.arange(b0, b0 + s.shape[1]) % 32) // 2
                sel = ((poly_mask >> pair) & 1).astype(bool)
                p[:, sel] = exp2_fma_pipe(x[:, sel])
            if skip_alpha_block == b0 // kbn:
                alpha = np.ones_like(alpha)
            m = mn
            l = (l * alpha + p.sum(axis=1, keepdims=True)).astype(ft)
            pv = (p.astype(np.float16).astype(ft) if kernel else p) @ v[b0:b0 + kbn].astype(ft)
            o = (o * alpha + pv).astype(ft)
    o = (o * (ft(1) / l)).astype(ft)
    if rms_g > 0:
        o = (o * (ft(rms_g) / np.sqrt((o * o).mean(axis=1, keepdims=True) + ft(1e-5)))).astype(ft)
    lse = ((m + np.log2(l)) * ft(math.log(2.0)))[:, 0]
    return (o.astype(np.float16) if kernel else o), lse
