"""fp64 reference, per-element error bound, input generators and a restatement of the host's tile choice for the fp8
(e4m3) scaled GEMM (b200_gemm_e4m3, hgemm.scaled_mm; csrc/gemm_fp8_sm90.cuh, csrc/gemm_fp8_capi.cu).

Kernel arithmetic, in order (K-blocks of 128, the last one zero-filled past K; an e4m3 zero is +0):
  1. the tensor core sums the 128 products of k-block j into a fresh accumulator, four k32 steps:  p_j ~ P_j
  2. promotion in fp32:   tensor / row   acc_j = fl32(acc_{j-1} + p_j)
                          block          acc_j = fl32(fma(p_j, g_j, acc_{j-1})),  g_j = fl32(sa[m, j] * sb[n // 128, j])
  3. epilogue scales:     tensor / row   v = fl32(fl32(acc * sa[m]) * sb[n])        block: v = acc
  4. one rounding to OutT (fp16 or bf16, round to nearest even)

Reference (`reference`).  Every product of two e4m3 values is exact in fp64 and so is every sum of 128 of them, so
P_j = sum_{k in block j} a_k b_k is exact.  C64 = sum_j g_j P_j (block; g_j is the fp32 product the kernel forms, taken
exactly) or sa sb sum_j P_j (tensor / row).  Alongside: S_j = sum_{k in block j} |a_k b_k| and
T_j = sum_{t=1..4} (|exact prefix of steps < t| bound + s_t) <= sum_{k in block j} (4 - (k mod 128) // 32) |a_k b_k|.

Bound (`bound`).  One named assumption, unmeasured (NVIDIA documents no precision for the e4m3 wgmma accumulation):

  TC(P)  each k32 step adds its 32 exact products to the accumulator with an error of at most
         2^-P (|acc| + sum |p|), P = 12 (DeepSeek-V3 reports about 14 bits retained on H800; 12 leaves margin).

With d = 2^-P and |acc| <= (1 + 4d) (prefix of |p|) inside a k-block, |p_j - P_j| <= d (1 + 4d) T_j (T_j as above:
step t sees the t - 1 earlier steps' magnitude plus its own).  Promotion adds at most u |acc_j| per k-block
(u = 2^-24, fp32), |acc_j| <= F sum_{i <= j} |g_i| S_i with F = (1 + 5d)(1 + u)^nkb, summed over j:
      E_acc = d (1 + 4d) sum_j |g_j| T_j + u F sum_i (nkb - i) |g_i| S_i          (g = 1 for tensor / row)
Tensor / row: the two epilogue products add (2u + u^2) |v|:  E = |sa sb| E_acc (1 + 2u + u^2) + (2u + u^2) |C64|.
Block: E = E_acc.  Then OutT's rounding (u_o = 2^-11 fp16, 2^-8 bf16; half a subnormal step h = 2^-25 fp16, 2^-134
bf16):
      |C - C64| <= u_o (|C64| + E) + E + h.
Nothing here is fitted to runs.  |C| below OutT's overflow threshold is assumed (fp16 overflow gives inf, by design).

Exact data (`int` generator, the probes, power-of-two scales): every in-block partial stays below 2^10 (128 products of
magnitude <= 4), which TC(P) reproduces exactly for any P >= 11, and every promoted sum, on the grid of its smallest
scale, stays below 2^24, so C before its rounding is exact and C = OutT(C64) bit for bit.
"""
from __future__ import annotations

import math

import numpy as np
import torch

E4 = torch.float8_e4m3fn
P_ASSUMED = 12                        # TC(P): stated, unmeasured
U32 = 2.0 ** -24
U_OUT = {torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8}
HALF_SUB = {torch.float16: 2.0 ** -25, torch.bfloat16: 2.0 ** -134}
BK = 128
RECIPES = ("tensor", "row", "block")
OUT_DTYPES = (torch.float16, torch.bfloat16)


# ------------------------------------------------------------------ e4m3
def _decode_code(c):
    s = -1.0 if c & 0x80 else 1.0
    e, m = (c >> 3) & 0xF, c & 0x7
    if e == 0xF and m == 0x7:
        return math.nan
    if e == 0:
        return s * m * 2.0 ** -9
    return s * (1 + m / 8) * 2.0 ** (e - 7)


E4M3_TABLE = np.array([_decode_code(c) for c in range(256)], dtype=np.float64)   # all 256 codes, fp64


def decode(x):
    """e4m3 tensor -> fp64 tensor, through the code table (independent of torch's own conversion)."""
    codes = x.contiguous().view(torch.uint8).long()
    return torch.from_numpy(E4M3_TABLE).to(x.device)[codes]


# ------------------------------------------------------------------ reference and bound
def kblocks(K):
    return -(-K // BK)


def block_scales(sa, sb, M, N, K):
    """g[j, m, n] = fl32(sa[m, j] * sb[n // 128, j]) as fp64, for the block recipe; sa [M, nkb], sb [nbs, nkb]."""
    g = sa.float().t()[:, :, None] * sb.float().t().repeat_interleave(BK, dim=1)[:, None, :N]
    return g.double()


def reference(a, b_nk, sa, sb, recipe, rows=None):
    """C64, E_acc terms and scales for C = scaled(A B^T).  a [M,K], b_nk [N,K] e4m3; sa, sb fp32 as the kernel reads
    them (tensor: one value each; row: [M], [N]; block: [M, nkb], [nbs, nkb]).  rows: sampled row indices or None."""
    A, B = decode(a), decode(b_nk)
    M, K = A.shape
    N = B.shape[0]
    ridx = torch.arange(M, device=A.device) if rows is None else torch.as_tensor(rows, device=A.device)
    A = A[ridx]
    nkb = kblocks(K)
    w = (4 - (torch.arange(K, device=A.device) % BK) // 32).double()
    c = torch.zeros(len(ridx), N, dtype=torch.float64, device=A.device)
    gt = torch.zeros_like(c)
    gs_weighted = torch.zeros_like(c)
    if recipe == "block":
        g_all = block_scales(sa.reshape(M, nkb)[ridx], sb.reshape(-1, nkb), len(ridx), N, K)
    for j in range(nkb):
        ks = slice(j * BK, min(K, (j + 1) * BK))
        Aj, Bj = A[:, ks], B[:, ks]
        P = Aj @ Bj.t()
        S = Aj.abs() @ Bj.abs().t()
        T = (Aj.abs() * w[ks]) @ Bj.abs().t()
        g = g_all[j] if recipe == "block" else 1.0
        c += g * P if recipe == "block" else P
        ag = abs(g) if recipe == "block" else 1.0
        gt += ag * T
        gs_weighted += (nkb - j) * ag * S
    d = 2.0 ** -P_ASSUMED
    F = (1 + 5 * d) * (1 + U32) ** nkb
    e_acc = d * (1 + 4 * d) * gt + U32 * F * gs_weighted
    ref = {"recipe": recipe, "nkb": nkb, "e_acc": e_acc, "rows": ridx}
    if recipe == "block":
        ref.update(c=c, e=e_acc)
    else:
        s_a = sa.double().reshape(-1)[ridx if recipe == "row" else torch.zeros_like(ridx)][:, None]
        s_b = sb.double().reshape(-1)[torch.arange(N, device=A.device) if recipe == "row" else
                                      torch.zeros(N, dtype=torch.long, device=A.device)][None, :]
        scale = s_a * s_b
        cs = c * scale
        e = scale.abs() * e_acc * (1 + 2 * U32 + U32 ** 2) + (2 * U32 + U32 ** 2) * cs.abs()
        ref.update(c=cs, e=e, unscaled=c, s_a=s_a, s_b=s_b)
    return ref


def bound(ref, out_dtype):
    return U_OUT[out_dtype] * (ref["c"].abs() + ref["e"]) + ref["e"] + HALF_SUB[out_dtype]


def rounded(ref, out_dtype):
    """OutT(C64): what exact data must produce bit for bit."""
    return ref["c"].float().to(out_dtype)


# ------------------------------------------------------------------ generators
GENERATORS = ("randn", "binade", "cancel", "k_probe", "a_probe", "int")
EXACT = ("k_probe", "a_probe", "int")
# e4m3 codes without NaN (0x7F, 0xFF) for the probes: distinct values along a row / column where possible
_FINITE_CODES = np.array([c for c in range(256) if c not in (0x7F, 0xFF, 0x00, 0x80)], dtype=np.uint8)


def _e4(x):
    return torch.as_tensor(x, dtype=torch.float32).to(E4)


def _from_codes(codes):
    return torch.from_numpy(np.ascontiguousarray(codes, dtype=np.uint8)).view(E4)


def make_inputs(gen, M, N, K, seed=0):
    """Seeded a [M,K] and b_nk [N,K] (e4m3, CPU) and probe data (or None).

    randn    torch.randn quantised with .to(float8_e4m3fn)
    binade   randn with row m of A scaled by 2^e_m, e in [-8, 2], and row n of B by 2^f_n, f in [-4, 2]: products
             span e4m3's subnormals up to 2^10
    cancel   the first half of k has positive A and B; the second half repeats A against a quantised -B + 2^-4 noise,
             so the running sum climbs to its maximum at K/2 and falls back: |C64| << s
    k_probe  B[n, k] = 1 iff k = sigma(n) (sigma reaches 0 and K - 1): C[m, n] = A[m, sigma(n)] exactly
    a_probe  A[m, k] = 1 iff k = tau(m): C[m, :] = B[:, tau(m)] exactly
    int      entries in {-2, ..., 2}: partials below 2^10, every promoted sum exact (see the module docstring)
    """
    g = torch.Generator().manual_seed(seed)
    rng = np.random.default_rng(seed)
    info = None
    if gen in ("randn", "binade"):
        a = torch.randn(M, K, generator=g)
        b = torch.randn(N, K, generator=g)
        if gen == "binade":
            a *= torch.exp2(torch.randint(-8, 3, (M, 1), generator=g).float())
            b *= torch.exp2(torch.randint(-4, 3, (N, 1), generator=g).float())
        return _e4(a), _e4(b), None
    if gen == "cancel":
        h = K // 2
        a = torch.randn(M, K, generator=g).abs()
        b = torch.randn(N, K, generator=g).abs()
        a[:, h:2 * h] = a[:, :h]
        b1 = _e4(b[:, :h]).float()
        b[:, :h] = b1
        b[:, h:2 * h] = -b1 + 2.0 ** -4 * torch.randn(N, h, generator=g)
        return _e4(a), _e4(b), None
    if gen == "int":
        return (_e4(torch.randint(-2, 3, (M, K), generator=g).float()),
                _e4(torch.randint(-2, 3, (N, K), generator=g).float()), None)
    if gen == "k_probe":
        sigma = rng.integers(0, K, N)
        sigma[0], sigma[-1] = K - 1, 0
        a = _FINITE_CODES[(np.arange(K)[None, :] + 131 * np.arange(M)[:, None]) % len(_FINITE_CODES)]
        b = np.zeros((N, K), np.float32)
        b[np.arange(N), sigma] = 1.0
        return _from_codes(a), _e4(b), {"sigma": sigma}
    if gen == "a_probe":
        tau = rng.integers(0, K, M)
        tau[0], tau[-1] = K - 1, 0
        a = np.zeros((M, K), np.float32)
        a[np.arange(M), tau] = 1.0
        b = _FINITE_CODES[(np.arange(K)[None, :] + 37 * np.arange(N)[:, None]) % len(_FINITE_CODES)]
        return _e4(a), _from_codes(b), {"tau": tau}
    raise ValueError(gen)


def make_scales(recipe, M, N, K, pow2, seed=0):
    """fp32 scales as the kernel reads them (tensor: [1], [1]; row: [M], [N]; block: [M, nkb] M-major storage, returned
    as the [M, nkb] view with stride (1, M), and [ceil(N/128), nkb] row-major).  pow2: powers of two in 2^-2 .. 2^2
    (exact data stays exact); else uniform in [0.25, 4), never 1."""
    g = torch.Generator().manual_seed(seed + 7)
    nkb, nbs = kblocks(K), -(-N // BK)

    def draw(*shape):
        if pow2:
            e = torch.randint(-2, 2, shape, generator=g).float()
            e = torch.where(e >= 0, e + 1, e)           # never 2^0
            return torch.exp2(e)
        x = torch.exp2(torch.rand(*shape, generator=g) * 4 - 2)
        return torch.where(x == 1, torch.full_like(x, 1.5), x)

    if recipe == "tensor":
        return draw(1), draw(1)
    if recipe == "row":
        return draw(M), draw(N)
    return draw(nkb, M).t(), draw(nbs, nkb)


# ------------------------------------------------------------------ restated arithmetic and its mutations (CPU)
def _tc_step(acc, step_sum, step_abs, P):
    """TC(P) realised: round the exact acc + step toward zero on the grid 2^(floor(log2(|acc| + sum|p|)) - P), an
    error below 2^-P (|acc| + sum|p|)."""
    exact = acc + step_sum
    mag = acc.abs() + step_abs
    ulp = torch.exp2(torch.floor(torch.log2(torch.where(mag > 0, mag, torch.ones_like(mag)))) - P)
    return torch.where(mag > 0, torch.trunc(exact / ulp) * ulp, exact)


def emulate(a, b_nk, sa, sb, recipe, out_dtype, P=P_ASSUMED, mutation=None, j_drop=None):
    """The kernel's arithmetic under TC(P), optionally with one mistake:
       drop_block     k-block j_drop is left out
       neighbour      row / tensor: row m uses row m+1's scale (mod M); block: k-block j uses block j+1's scales
       no_epi_scale   tensor / row: sb is never applied; block: the weight scale sb is left out of g
       second_round   the promoted sum rounded to OutT after every k-block (C accumulated in OutT)
       no_promotion   tensor / row: one tensor-core accumulator over the whole K (scale-d = 0 only at k = 0)
    Returns OutT C as fp64 [M, N]."""
    A, B = decode(a), decode(b_nk)
    M, K = A.shape
    N = B.shape[0]
    nkb = kblocks(K)
    Ap = torch.zeros(M, nkb * BK, dtype=torch.float64)
    Bp = torch.zeros(N, nkb * BK, dtype=torch.float64)
    Ap[:, :K], Bp[:, :K] = A, B
    acc = torch.zeros(M, N, dtype=torch.float32)
    tc = torch.zeros(M, N, dtype=torch.float64)
    if recipe == "block":
        sa_use = sa.reshape(M, nkb)
        sb_use = sb.reshape(-1, nkb)
        if mutation == "no_epi_scale":
            sb_use = torch.ones_like(sb_use)
        g_all = block_scales(sa_use, sb_use, M, N, K)
        if mutation == "neighbour":
            g_all = g_all[(torch.arange(nkb) + 1) % nkb]
    for j in range(nkb):
        if mutation != "no_promotion" or j == 0:
            tc = torch.zeros(M, N, dtype=torch.float64)
        for t in range(4):
            ks = slice(j * BK + 32 * t, j * BK + 32 * t + 32)
            Aj, Bj = Ap[:, ks], Bp[:, ks]
            tc = _tc_step(tc, Aj @ Bj.t(), Aj.abs() @ Bj.abs().t(), P)
        if mutation == "drop_block" and j == j_drop:
            continue
        p = tc.float()
        if mutation == "no_promotion":
            continue
        if recipe == "block":
            acc = (p.double() * g_all[j].float().double() + acc.double()).float()   # fma: one rounding
        else:
            acc = acc + p
        if mutation == "second_round":
            acc = acc.to(out_dtype).float()
    if mutation == "no_promotion":
        acc = tc.float()
    if recipe == "block":
        return acc.to(out_dtype).double()
    s_a = sa.float().reshape(-1)
    s_b = sb.float().reshape(-1)
    s_a = s_a.expand(M) if recipe == "tensor" else s_a
    s_b = s_b.expand(N) if recipe == "tensor" else s_b
    if mutation == "neighbour":
        s_a = s_a[(torch.arange(M) + 1) % M]
    if mutation == "no_epi_scale":
        s_b = torch.ones_like(s_b)
    v = (acc * s_a[:, None]) * s_b[None, :]
    return v.to(out_dtype).double()


# ------------------------------------------------------------------ tile choice (gemm_fp8_capi.cu) and instantiations
BM, BN, GROUP_M, STAGES = 128, 128, 16, 6
SMS = 132                       # H100 SXM
CLUSTER_SLOTS = 66              # at most SMS / 2 clusters of two at once (cudaOccupancyMaxActiveClusters decides)


def tile_plan(M, N, K):
    """The host's launch, restated: 128 x 128 tiles, clusters of two CTAs whenever there are two m-tiles, cluster tiles
    walked in raster groups of 16 m-tiles (8 pairs), one k-block per 128 of K."""
    tm, tn = -(-M // BM), -(-N // BN)
    cs = 2 if tm >= 2 else 1
    rows = -(-tm // cs)
    num_tiles = rows * tn
    group = GROUP_M // cs
    slots = CLUSTER_SLOTS if cs == 2 else SMS
    clusters = min(num_tiles, slots)
    return {"tiles_m": tm, "tiles_n": tn, "cs": cs, "num_tiles": num_tiles, "clusters": clusters,
            "tiles_per_cluster": -(-num_tiles // clusters), "kblocks": kblocks(K),
            "groups": [(g * group, min(group, rows - g * group)) for g in range(-(-rows // group))],
            "odd_tiles_m": tm % 2 == 1 and tm > 1}


INSTANTIATIONS = [("__half", False), ("__half", True), ("__nv_bfloat16", False), ("__nv_bfloat16", True)]
OUT_NAME = {torch.float16: "__half", torch.bfloat16: "__nv_bfloat16"}


def instantiation(out_dtype, recipe):
    """gemm_e4m3_kernel<OutT, kBlockScale> of a call: tensor and row share kBlockScale = false."""
    return (OUT_NAME[out_dtype], recipe == "block")


def parse_instantiations(names):
    """(OutT, kBlockScale) of every gemm_e4m3_kernel name, mangled or demangled."""
    out = []
    for n in names:
        if "gemm_e4m3_kernel" not in n:
            continue
        t = "__nv_bfloat16" if "bfloat16" in n else "__half"
        if "Lb1E" in n or "true>" in n:
            blk = True
        elif "Lb0E" in n or "false>" in n:
            blk = False
        else:
            continue
        out.append((t, blk))
    return out


# GPU shape table: (M, N, K) -> what it reaches.  Every recipe x OutT runs every shape.
SHAPES = [
    (1, 8, 16),          # M = 1, N = 8, K below one k-block; one CTA, no cluster
    (77, 136, 48),       # ragged M, N, K inside one m-tile; two n-tiles, the second 8 columns wide
    (200, 264, 208),     # one cluster pair, the rank-1 m-tile ragged; K = one block + a ragged one
    (385, 520, 400),     # odd tiles_m = 4 -> two pairs; ragged everything
    (2600, 2344, 512),   # tiles_m 21 (odd, last pair half past M), raster groups of 8 + 3 pairs, > 1 tile per cluster
    (4096, 4096, 64),    # 512 single-k-block cluster tiles, 8 per cluster: the 6-stage ring wraps across tiles
    (640, 392, 4096),    # 32 k-blocks per tile
]
