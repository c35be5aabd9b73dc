"""KV-cache append with rotary embedding (b200_kvcache_append_{f16,bf16}[_paged], flash_attn.kvcache_append and
flash_attn.fmha_fwd_kvcache) restated on the CPU: where each new token goes, the two rotary pairings against fp64 with
their bound, the e4m3 rule, the expected cache after an append, the kernel's arithmetic (for the sharpness tests) and the
GPU case table.  Used by test_kvcache_args.py, test_kvcache_sharpness.py, test_kvcache_coverage.py and
test_kvcache_gpu.py.

Positions.  Sequence b holds L_b = clamp(cache_seqlens[b], 0, capacity) tokens; new token t goes to p = L_b + t.  Dense
[B, Hkv, Nk, D] caches (capacity Nk): row p of (b, h).  Paged pools [num_pages, page_size, Hkv, D] (capacity
max_pages * page_size): row p % page_size of page table[b][p // page_size].  Not written: p >= capacity, and a table
entry outside [0, num_pages).  q is rotated at p for every token.  seqlens_out[b] = min(L_b + n_new, capacity).

Rotary.  Pair i is (2i, 2i+1) interleaved (GPT-J), else (i, i + rotary_dim / 2) (NeoX); x0' = x0 c - x1 s,
x1' = x0 s + x1 c with c, s = cos[p, i], sin[p, i] (fp32 tables).  The kernel computes one product rounded to fp32 and
the other fused (two fp32 roundings, each <= 2^-24 of a term no larger than |x0 c| + |x1 s|), then rounds once to T:
  |x' - exact| <= ulp_T(exact) + 2^-22 (|x0 c| + |x1 s|)      (for x1': |x0 s| + |x1 c|)
ulp_T(y) is T's spacing at |y| (its smallest spacing below the normal range): the rounding to T moves the fp32 value
by at most half its spacing, which is at most the spacing at |exact| once the fp32 error is accounted for.  Columns past
rotary_dim are copied, so they and every v row are exact.

e4m3.  A cache code is (x_T.float() / scale).clamp(-448, 448).to(float8_e4m3fn), x_T the T value after rotary.  torch's
own conversion turns overflow into NaN, hence the clamp; the kernel's cvt.rn.satfinite saturates.
"""
from __future__ import annotations

import re
from collections import namedtuple

import numpy as np
import torch

TYPES = ("half", "bf16")
TORCH = {"half": torch.float16, "bf16": torch.bfloat16}
MANT = {"half": 10, "bf16": 7}                  # stored mantissa bits
MIN_SPACING = {"half": 2.0 ** -24, "bf16": 2.0 ** -133}
MIN_NORMAL_EXP = {"half": -14, "bf16": -126}
CACHES = ("T", "e4m3")
LAYOUTS = ("dense", "paged")
ROTARY = ("none", "interleaved", "neox", "partial")
E4M3_MAX = 448.0
REL = 2.0 ** -22


# ------------------------------------------------------------------ positions
def clamp_len(L, capacity):
    return min(max(int(L), 0), capacity)


def slot(b, t, L, capacity, table=None, page_size=None, num_pages=None):
    """Where token t of sequence b goes: a dense position p, a paged (page, row), or None when it is not written."""
    p = clamp_len(L, capacity) + t
    if p >= capacity:
        return None
    if table is None:
        return p
    page = int(table[b][p // page_size])
    if not 0 <= page < num_pages:
        return None
    return page, p % page_size


def seqlens_out(lens, n_new, capacity):
    return [min(clamp_len(L, capacity) + n_new, capacity) for L in lens]


def cache_rows(B, Hkv, n_new, lens, capacity, table=None, page_size=None, num_pages=None):
    """(src, dst) int64 tensors over the rows of k_new viewed as [B * Hkv * n_new, D] and of the cache viewed as
    [rows, D]: every row the append writes."""
    src, dst = [], []
    for b in range(B):
        for t in range(n_new):
            s = slot(b, t, lens[b], capacity, table, page_size, num_pages)
            if s is None:
                continue
            for h in range(Hkv):
                src.append((b * Hkv + h) * n_new + t)
                if table is None:
                    dst.append((b * Hkv + h) * capacity + s)
                else:
                    dst.append((s[0] * page_size + s[1]) * Hkv + h)
    return torch.tensor(src, dtype=torch.int64), torch.tensor(dst, dtype=torch.int64)


def positions(B, heads, n_new, lens, capacity):
    """[B * heads * n_new] int64: the position of every row of a [B, heads, n_new, D] tensor."""
    p = torch.tensor([[clamp_len(lens[b], capacity) + t for t in range(n_new)] for b in range(B)], dtype=torch.int64)
    return p[:, None, :].expand(B, heads, n_new).reshape(-1)


# ------------------------------------------------------------------ rotary
def tables(rotary_len, rotary_dim, base=10000.0):
    """fp32 cos, sin [rotary_len, rotary_dim / 2] of angle p * base^(-2i / rotary_dim)."""
    inv = 1.0 / base ** (np.arange(0, rotary_dim, 2, dtype=np.float64) / rotary_dim)
    ang = np.arange(rotary_len, dtype=np.float64)[:, None] * inv[None, :]
    return torch.from_numpy(np.cos(ang).astype(np.float32)), torch.from_numpy(np.sin(ang).astype(np.float32))


def pair_index(D, rotary_dim, interleaved):
    """(i0, i1) column index arrays of the pairs: x0 = x[..., i0], x1 = x[..., i1], pair k uses table column k."""
    k = np.arange(rotary_dim // 2)
    return (2 * k, 2 * k + 1) if interleaved else (k, k + rotary_dim // 2)


def rotate_exact(x, cos, sin, pos, rotary_dim, interleaved):
    """(fp64 rotated rows, fp64 magnitude term per element) of rows x [R, D] (any float type) at positions pos [R]:
    the exact rotation of the stored values and |x0 c| + |x1 s| (resp. |x0 s| + |x1 c|); columns past rotary_dim
    are the input with magnitude 0."""
    x = x.double()
    out, mag = x.clone(), torch.zeros_like(x)
    if rotary_dim == 0:
        return out, mag
    i0, i1 = pair_index(x.shape[1], rotary_dim, interleaved)
    c, s = cos.double()[pos], sin.double()[pos]
    x0, x1 = x[:, i0], x[:, i1]
    out[:, i0], out[:, i1] = x0 * c - x1 * s, x0 * s + x1 * c
    mag[:, i0], mag[:, i1] = (x0 * c).abs() + (x1 * s).abs(), (x0 * s).abs() + (x1 * c).abs()
    return out, mag


def ulp(y, T):
    """T's spacing at |y| (fp64 tensor), its smallest spacing below the normal range."""
    a = y.abs()
    e = torch.floor(torch.log2(torch.where(a > 0, a, torch.ones_like(a))))
    e = torch.clamp(e, min=MIN_NORMAL_EXP[T])
    return torch.where(a > 0, torch.pow(2.0, e - MANT[T]), torch.full_like(a, MIN_SPACING[T]))


def bound(exact, mag, T):
    """Per-element bound of the kernel's rotated T value against the exact rotation (0 where nothing is rotated)."""
    return torch.where(mag > 0, ulp(exact, T) + REL * mag, torch.zeros_like(mag))


def within(got, exact, mag, T):
    """bool tensor: got (T values) within the rotary bound of the exact rotation; unrotated columns must be equal."""
    return (got.double() - exact).abs() <= bound(exact, mag, T)


# ------------------------------------------------------------------ e4m3
def quantise(x, scale):
    """The cache codes of T values x: (x.float() / scale).clamp(-448, 448) in e4m3, round to nearest even."""
    return (x.float() / scale).clamp(-E4M3_MAX, E4M3_MAX).to(torch.float8_e4m3fn)


# ------------------------------------------------------------------ the kernel's arithmetic
def _f32(x):
    return np.asarray(x, np.float64).astype(np.float32).astype(np.float64)


def kernel_rotate(x, cos, sin, pos, rotary_dim, interleaved, T, mistake=None):
    """The kernel's rotary on rows x [R, D] of T values (torch), as a T tensor: x0' = fma(x0, c, -fp32(x1 s)),
    x1' = fma(x0, s, fp32(x1 c)), rounded once to T.  The fma is exact in fp64 (a T value times an fp32 value has at
    most 35 significant bits) before its rounding to fp32, up to the fp64 rounding of the sum (far below 2^-24).
    `mistake` injects one wrong design: "pairing" (the other pairing), "position" (rotated at p + 1), "swap" (cos and
    sin exchanged)."""
    if rotary_dim == 0:
        return x.clone()
    if mistake == "pairing":
        interleaved = not interleaved
    if mistake == "position":
        pos = pos + 1
    if mistake == "swap":
        cos, sin = sin, cos
    xd = x.double().numpy()
    out = xd.copy()
    i0, i1 = pair_index(x.shape[1], rotary_dim, interleaved)
    c, s = cos.double().numpy()[pos.numpy()], sin.double().numpy()[pos.numpy()]
    x0, x1 = xd[:, i0], xd[:, i1]
    out[:, i0] = _f32(x0 * c - _f32(x1 * s))
    out[:, i1] = _f32(x0 * s + _f32(x1 * c))
    return torch.from_numpy(out).to(torch.float32).to(TORCH[T])


def kernel_quantise(x, scale, mistake=None):
    """The kernel's e4m3 store of T values x; mistakes "multiply" (x * (1 / scale)) and "no_saturation" (torch's
    conversion without the clamp: overflow becomes NaN)."""
    if mistake == "multiply":
        return (x.float() * np.float32(1.0 / scale)).clamp(-E4M3_MAX, E4M3_MAX).to(torch.float8_e4m3fn)
    if mistake == "no_saturation":
        return (x.float() / scale).to(torch.float8_e4m3fn)
    return quantise(x, scale)


def kernel_append(cache, new, lens, capacity, cos, sin, rotary_dim, interleaved, T, scale=1.0, table=None,
                  page_size=None, num_pages=None, rotate=True, mistake=None):
    """The cache (a [rows, D] view of dense or paged storage, T or float8_e4m3fn, modified in place) after the kernel's
    append of new [B, Hkv, n_new, D] (T); rotate=False for v.  `mistake` may also be "early": every token written one
    row before its slot."""
    B, Hkv, n_new, D = new.shape
    src, dst = cache_rows(B, Hkv, n_new, lens, capacity, table, page_size, num_pages)
    if src.numel() == 0:
        return cache
    rows = new.reshape(-1, D)[src]
    if rotate:
        pos = positions(B, Hkv, n_new, lens, capacity)[src]
        rows = kernel_rotate(rows, cos, sin, pos, rotary_dim, interleaved, T, mistake)
    if cache.dtype == torch.float8_e4m3fn:
        rows = kernel_quantise(rows, scale, mistake)
    if mistake == "early":
        dst = dst - (1 if table is None else Hkv)
        keep = dst >= 0
        dst, rows = dst[keep], rows[keep]
    cache[dst] = rows
    return cache


def check_append(after, before, new, lens, capacity, cos, sin, rotary_dim, interleaved, T, scale=1.0, table=None,
                 page_size=None, num_pages=None, rotate=True):
    """None if `after` (a [rows, D] cache view, CPU) is `before` with exactly the restated append, else the first
    violation as text.  T caches: touched rows bit for bit without rotary, within the bound with it; e4m3 caches: the
    codes of a T value within the bound (without rotary: exactly quantise of the new rows); every other row bit for bit
    `before`."""
    B, Hkv, n_new, D = new.shape
    src, dst = cache_rows(B, Hkv, n_new, lens, capacity, table, page_size, num_pages)
    e4m3 = after.dtype == torch.float8_e4m3fn
    raw = (lambda x: x.view(torch.uint8)) if e4m3 else (lambda x: x.view(torch.int16))
    untouched = torch.ones(after.shape[0], dtype=torch.bool)
    untouched[dst] = False
    if not torch.equal(raw(after)[untouched], raw(before)[untouched]):
        return "a row the append does not own changed"
    if src.numel() == 0:
        return None
    rows = new.reshape(-1, D)[src]
    got = after[dst]
    rot = rotate and rotary_dim > 0
    if not rot:
        want = quantise(rows, scale) if e4m3 else rows
        return None if torch.equal(raw(got), raw(want)) else "a written row differs from the new row"
    pos = positions(B, Hkv, n_new, lens, capacity)[src]
    exact, mag = rotate_exact(rows, cos, sin, pos, rotary_dim, interleaved)
    if e4m3:
        # every code the bound allows: the codes of the extreme T values in [exact - bound, exact + bound]
        b = bound(exact, mag, T)
        lo = quantise((exact - b).to(TORCH[T]), scale).float()
        hi = quantise((exact + b).to(TORCH[T]), scale).float()
        g = got.float()
        ok = (g >= torch.minimum(lo, hi)) & (g <= torch.maximum(lo, hi))
        return None if bool(ok.all()) else "a written e4m3 code lies outside the rotary bound"
    return None if bool(within(got, exact, mag, T).all()) else "a written row lies outside the rotary bound"


# ------------------------------------------------------------------ instantiations
def instantiation(T, cache):
    """The kernel template arguments (T, CacheT) of a call with element type T and cache "T" or "e4m3"."""
    return (T, T if cache == "T" else "e4m3")


INSTANTIATIONS = sorted({instantiation(T, c) for T in TYPES for c in CACHES})
_NAMES = {"half": "__half", "bf16": "__nv_bfloat16", "e4m3": "__nv_fp8_e4m3"}
_MANGLED = re.compile(r"kvcache_append_kernelI(6__half|13__nv_bfloat16)(S1_|13__nv_fp8_e4m3)E")
_DEMANGLED = re.compile(r"kvcache_append_kernel<(__half|__nv_bfloat16), (__half|__nv_bfloat16|__nv_fp8_e4m3)>")
_FROM = {"6__half": "half", "13__nv_bfloat16": "bf16", "__half": "half", "__nv_bfloat16": "bf16",
         "13__nv_fp8_e4m3": "e4m3", "__nv_fp8_e4m3": "e4m3"}


def name(inst):
    return f"kvcache_append_kernel<{_NAMES[inst[0]]}, {_NAMES[inst[1]]}>"


def parse_instantiations(names):
    out = []
    for n in names:
        for m in _MANGLED.finditer(n):
            t = _FROM[m.group(1)]
            out.append((t, t if m.group(2) == "S1_" else _FROM[m.group(2)]))
        for m in _DEMANGLED.finditer(n):
            out.append((_FROM[m.group(1)], _FROM[m.group(2)]))
    return out


# ------------------------------------------------------------------ the GPU case table
# rotary: "none", "interleaved" / "neox" over every column, "partial" NeoX over half of them (a multiple of 16)
Case = namedtuple("Case", "T cache layout rotary D n_new page_size lens table_kind")
# lens are chosen against a capacity of 512 positions (dense Nk = 512; paged 512 / page_size pages per sequence): they
# include empty sequences, one clamped from below (-5), one that overflows, and one past capacity.
LENS = {1: [0, 37, 511, 512, 700, -5], 4: [0, 37, 510, 300, 2000, -5], 130: [0, 200, 400, 129, 600, 31]}
CAPACITY = 512


def rotary_dim(c):
    return {"none": 0, "interleaved": c.D, "neox": c.D, "partial": (c.D // 2) // 16 * 16 or 16}[c.rotary]


def _cases():
    dims = (64, 128, 256, 80)
    news = (1, 4, 130)
    out = []
    i = 0
    for T in TYPES:
        for cache in CACHES:
            for layout in LAYOUTS:
                for rot in ROTARY:
                    D = dims[(i + i // 4) % 4]
                    n_new = news[i % 3]
                    ps = (16, 256)[(i + i // 4) % 2] if layout == "paged" else None
                    table_kind = ("bad" if (i // 2) % 2 else "good") if layout == "paged" else None
                    out.append(Case(T, cache, layout, rot, D, n_new, ps, LENS[n_new], table_kind))
                    i += 1
    return out


CASES = _cases()


def combo(c):
    return (c.T, c.cache, c.layout, c.rotary)


def combos():
    return {(T, c, l, r) for T in TYPES for c in CACHES for l in LAYOUTS for r in ROTARY}


# the shapes of tools/bench_kvcache.py (test_kvcache_coverage checks that they agree):
# (name, B, H, Hkv, D, n_new, page_size, cache) for decode steps; (name, B, Hkv, D, n_new, cache) for appends
BENCH_DECODE = [("decode p16 fp16", 32, 32, 8, 128, 1, 16, "fp16"), ("decode p256 fp16", 32, 32, 8, 128, 1, 256, "fp16"),
                ("decode p16 e4m3", 32, 32, 8, 128, 1, 16, "e4m3"), ("decode p256 e4m3", 32, 32, 8, 128, 1, 256, "e4m3")]
BENCH_APPEND = [("prefill append fp16", 4, 8, 128, 2048, "fp16"), ("prefill append e4m3", 4, 8, 128, 2048, "e4m3")]
BENCH_LK_RANGE = (256, 8192)


def bench_lengths(B, seed):
    rng = np.random.default_rng(seed)
    return [int(x) for x in rng.integers(BENCH_LK_RANGE[0], BENCH_LK_RANGE[1] + 1, size=B)]


def append_bytes(B, Hkv, D, n_new, cache, H=0):
    """Bytes an append reads and writes: k, v (and q, read and written) in fp16, the cache rows in fp16 or e4m3."""
    elems = B * Hkv * n_new * D
    return 2 * elems * 2 + 2 * elems * (1 if cache == "e4m3" else 2) + 2 * B * H * n_new * D * 2
