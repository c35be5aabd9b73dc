"""Every entry family past 2^31 elements / 2^32 bytes and at B * Hkv = 65535, on the GPU (the case table: large_ref.py).

Per case:
  * skipped, with the numbers, when the device has less free memory than the restated peak plus a margin;
  * torch.cuda.max_memory_allocated() during the call against the restated peak;
  * NaN guard bands after every output (and NaN-poisoned outputs), checked after the call;
  * _capi.launch_count() up by the launches of the intended path;
  * two oracles: the same entry point on a small slice of the same data, bit for bit (rows and heads are independent;
    the slices are the first, the one straddling 2^31 elements and the last), and the fp64 references of the other
    test modules with their per-element bounds on sampled rows, built in chunks on the device;
  * its tensors freed and the cache emptied before the next case.
The measured peaks are printed ("[large] ...") for the record.
"""
from __future__ import annotations

import gc
import math

import pytest
import torch

import attn_bf16_ref as BF
import attn_fp8kv_ref as F8
import attn_paged_ref as PG
import attn_ref as R
import attn_seqlens_ref as S
import attn_split_ref as SR
import gemm_ref as G
import large_ref as L
import merge_ref as MR
import rope_rms_ref as RR
from leetcuda_b200 import _capi, flash_attn, fused_ops, hgemm, merge_attn_states, rms_norm, rope, sgemm

MARGIN = 2 * L.GiB                     # the oracles' own tensors
PEAK_SLACK = 8 * 2 ** 20               # the allocator rounds each tensor up (to 512 bytes, a large one by < 2 MiB)
BASE_LIMIT = 64 * 2 ** 20              # what torch keeps between cases (the cuBLAS workspace of the fp64 oracles)
_BASE = [0]                            # bytes allocated before the case's own tensors
TORCH = {"f16": torch.float16, "bf16": torch.bfloat16, "f32": torch.float32}
dev = "cuda"


# ------------------------------------------------------------------ harness
def guarded(shape, dtype):
    """(view of shape, flat buffer): NaN everywhere, GUARD NaN elements past the view."""
    n = math.prod(shape)
    buf = torch.full((n + L.GUARD,), float("nan"), dtype=dtype, device=dev)
    return buf[:n].view(shape), buf


def guard_intact(buf, n, what):
    g = buf[n:]
    assert torch.isnan(g.float()).all(), f"{what}: the guard band after the output was written"


def randn(shape, dtype, seed):
    gen = torch.Generator(device=dev).manual_seed(seed)
    return torch.randn(shape, dtype=dtype, device=dev, generator=gen)


class Run:
    """Counts the launches and the peak of torch allocations of one call."""

    def __init__(self, case):
        self.case = case

    def __enter__(self):
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()     # from the inputs' allocation on: what the call adds
        self.n0 = _capi.launch_count()
        return self

    def __exit__(self, *exc):
        torch.cuda.synchronize()
        self.launches = _capi.launch_count() - self.n0
        self.peak = torch.cuda.max_memory_allocated()
        return False


def check_peak(case, peak):
    peak -= _BASE[0]
    print(f"[large] {case.name}: peak {peak / L.GiB:.3f} GiB measured, {case.peak / L.GiB:.3f} GiB restated"
          f" (+ {case.scratch / L.GiB:.3f} GiB library scratch)")
    assert abs(peak - case.peak) <= PEAK_SLACK, (case.name, peak, case.peak)


def same(a, b, what):
    assert a.shape == b.shape, what
    eq = (a == b) | (torch.isnan(a.float()) & torch.isnan(b.float()))
    assert bool(eq.all()), f"{what}: {int((~eq).sum())} elements differ from the sliced call"


def within(got, want, bound, what):
    err = (got.double() - want).abs()
    bad = ~(err <= bound)
    assert not bool(bad.any()), (f"{what}: {int(bad.sum())} elements out of bound, worst excess "
                                 f"{float((err - bound)[bad].max())}")


# ------------------------------------------------------------------ attention
def _attn_fp64(o, lse, q, k, v, causal, lq, lk, dtype, what):
    """One batch: o, lse [1, H, Nq(, D)], q [1, H, Nq, D], k, v [1, Hkv, Nk, D] against attn_seqlens_ref."""
    D = q.shape[-1]
    poly = D <= 128
    ref = S.reference(q, k, v, R.kernel_scale(D), causal, [lq], [lk])
    ob = (BF.o_bound(ref, poly) if dtype == "bf16" else R.o_bound(ref, poly))[1]
    within(o, ref["o"], ob, what + " O")
    live = ~ref["empty"]
    lb = R.lse_bound(ref, poly)
    within(lse[live], ref["lse"][live], lb[live], what + " lse")
    assert bool(torch.isneginf(lse[~live]).all()), what + " lse of empty rows"


def _dense_call(c, q, k, v, o, lse, lq=None, lk=None):
    s = c.shape
    flash_attn.fmha_fwd(q, k, v, o, lse=lse, causal=s["causal"], num_splits=s.get("splits", 1),
                        seqlens_q=lq, seqlens_k=lk, k_scale=s.get("k_scale", 1.0), v_scale=s.get("v_scale", 1.0))


def _batch_slices(B, per_batch):
    cross = L.TWO31 // per_batch
    return sorted({0, min(cross, B - 1), B - 1})


def run_dense(c):
    s = c.shape
    T = TORCH[c.dtype]
    B, H, Hkv, Nq, Nk, D = s["B"], s["H"], s["Hkv"], s["Nq"], s["Nk"], s["D"]
    fp8 = s.get("kv") == "e4m3"
    q = randn((B, H, Nq, D), T, 1)
    if fp8:
        k, v = _fp8_codes((B, Hkv, Nk, D), 2), _fp8_codes((B, Hkv, Nk, D), 3)
    else:
        k, v = randn((B, Hkv, Nk, D), T, 2), randn((B, Hkv, Nk, D), T, 3)
    o, ob = guarded((B, H, Nq, D), T)
    lse, lb = guarded((B, H, Nq), torch.float32)
    lens = None
    if "lq" in s:
        lens = (torch.tensor(s["lq"], dtype=torch.int32, device=dev), torch.tensor(s["lk"], dtype=torch.int32, device=dev))
    with Run(c) as r:
        if lens:
            _dense_call(c, q, k, v, o, lse, *lens)
        else:
            _dense_call(c, q, k, v, o, lse)
    check_peak(c, r.peak)
    assert r.launches == (2 if s.get("splits", 1) > 1 else 1), r.launches
    guard_intact(ob, o.numel(), c.name + " O")
    guard_intact(lb, lse.numel(), c.name + " lse")
    for b in _batch_slices(B, max(H * Nq * D, Hkv * Nk * D)):
        so, sl = torch.empty_like(o[b:b + 1]), torch.empty_like(lse[b:b + 1])
        if lens:
            _dense_call(c, q[b:b + 1], k[b:b + 1], v[b:b + 1], so, sl, lens[0][b:b + 1], lens[1][b:b + 1])
        else:
            _dense_call(c, q[b:b + 1], k[b:b + 1], v[b:b + 1], so, sl)
        same(o[b:b + 1], so, f"{c.name} O batch {b}")
        same(lse[b:b + 1], sl, f"{c.name} lse batch {b}")
        lq = s["lq"][b] if lens else Nq
        lk = s["lk"][b] if lens else Nk
        if s.get("splits", 1) > 1:
            _split_fp64(c, o[b:b + 1], lse[b:b + 1], q[b:b + 1], k[b:b + 1], v[b:b + 1], b)
        elif fp8:
            _fp8_fp64(o[b:b + 1], lse[b:b + 1], q[b:b + 1], k[b:b + 1].float(), v[b:b + 1].float(), c, lq, lk,
                      f"{c.name} batch {b}")
        else:
            _attn_fp64(o[b:b + 1], lse[b:b + 1], q[b:b + 1], k[b:b + 1], v[b:b + 1], s["causal"], lq, lk, c.dtype,
                       f"{c.name} batch {b}")


def _split_fp64(c, o, lse, q, k, v, b):
    """Non-causal split rows: the parts are the key-block ranges of attn_split_ref.split_ranges; sampled query rows."""
    s = c.shape
    Nk, D, G = s["Nk"], s["D"], s["H"] // s["Hkv"]
    kbn = R.family(D)[1]
    rows = torch.cat([torch.arange(0, 32), torch.arange(s["Nq"] - 32, s["Nq"])]).to(dev)
    qs = q[:, :, rows]
    ke, ve = SR.expand(k, G), SR.expand(v, G)
    parts = []
    for lo, hi in SR.split_ranges((Nk + kbn - 1) // kbn, s["splits"]):
        vis = torch.zeros(len(rows), Nk, dtype=torch.bool, device=dev)
        vis[:, lo * kbn:min(hi * kbn, Nk)] = True
        parts.append(SR.masked_reference(qs, ke, ve, R.kernel_scale(D), vis[None, None]))
    want, L_, empty, obnd, lbnd = SR.combine_bound(parts, D <= 128)
    within(o[:, :, rows], want, obnd, f"{c.name} batch {b} O")
    within(lse[:, :, rows], L_, lbnd, f"{c.name} batch {b} lse")


def run_rms(c):
    s = c.shape
    B, H, N, D, g = s["B"], s["H"], s["Nq"], s["D"], s["g"]
    q, k, v = (randn((B, H, N, D), torch.float16, i) for i in (11, 12, 13))
    o, ob = guarded((B, H, N, D), torch.float16)
    with Run(c) as r:
        fused_ops.attn_rmsnorm(q, k, v, o, g)
    check_peak(c, r.peak)
    assert r.launches == 1
    guard_intact(ob, o.numel(), c.name)
    for b in _batch_slices(B, H * N * D):
        so = torch.empty_like(o[b:b + 1])
        fused_ops.attn_rmsnorm(q[b:b + 1], k[b:b + 1], v[b:b + 1], so, g)
        same(o[b:b + 1], so, f"{c.name} batch {b}")
        for h in (0, H - 1):
            ref = R.reference(q[b, h], k[b, h], v[b, h], R.kernel_scale(D))
            y, yb = R.rms_reference(ref, g, R.o_bound(ref, D <= 128)[0])
            within(o[b, h], y, yb, f"{c.name} batch {b} head {h}")


def run_long(c):
    """The keys past 2^31 elements of K (rows >= tail) carry the softmax: q ~ 1 + 0.25 randn, tail keys ~ 9 + 0.5 randn
    score ~100 above the rest (randn keys, |score| < ~6), so every other key's weight is below e^-90 and O is the
    weighted mean of the tail's V rows (4 + randn).  A misread tail key moves O by O(|V|).  The same call on a copy of
    the tail alone, at a fresh base with small offsets, must then give the same O and lse bit for bit: the other keys
    only feed a running max and sum that the tail's first block rescales by ex2(-~100) = 0 (no effect in fp32)."""
    s = c.shape
    H, Nk, D, tail = s["H"], s["Nk"], s["D"], s["tail"]
    gen = torch.Generator(device=dev).manual_seed(21)
    q = (1 + 0.25 * torch.randn((1, H, 1, D), device=dev, generator=gen)).half()
    k = randn((1, 1, Nk, D), torch.float16, 22)
    v = randn((1, 1, Nk, D), torch.float16, 23)
    n = Nk - tail
    k[0, 0, tail:] = (9 + 0.5 * torch.randn((n, D), device=dev, generator=gen)).half()
    v[0, 0, tail:] = (4 + torch.randn((n, D), device=dev, generator=gen)).half()
    outs = {}
    for sp in s["splits"]:
        outs[sp] = guarded((1, H, 1, D), torch.float16) + guarded((1, H, 1), torch.float32)
    with Run(c) as r:
        counts = []
        for sp in s["splits"]:
            o, _, lse, _ = outs[sp]
            n0 = _capi.launch_count()
            flash_attn.fmha_fwd(q, k, v, o, lse=lse, num_splits=sp)
            counts.append(_capi.launch_count() - n0)
    check_peak(c, r.peak)
    assert counts == [1 if sp == 1 else 2 for sp in s["splits"]], counts
    ref = _long_reference(q[0, :, 0], k[0, 0], v[0, 0], R.kernel_scale(D))
    # the tail carries the weight: O is the tail's mean, far from the mean of the other rows of V
    assert float(ref["o"].min()) > 3.0, "the keys past 2^31 elements do not dominate the softmax"
    ob = R.o_bound(ref, True)[1]
    lbd = R.lse_bound(ref, True)
    kt, vt = k[:, :, tail:].clone(), v[:, :, tail:].clone()
    to, tl = torch.empty_like(outs[1][0]), torch.empty_like(outs[1][2])
    flash_attn.fmha_fwd(q, kt, vt, to, lse=tl, num_splits=1)
    for sp in s["splits"]:
        o, obuf, lse, lbuf = outs[sp]
        guard_intact(obuf, o.numel(), f"{c.name} splits {sp} O")
        guard_intact(lbuf, lse.numel(), f"{c.name} splits {sp} lse")
        same(o, to, f"{c.name} splits {sp}: O against the call on the tail keys alone")
        same(lse, tl, f"{c.name} splits {sp}: lse against the call on the tail keys alone")
        within(o[0, :, 0], ref["o"], ob, f"{c.name} splits {sp} O")
        within(lse[0, :, 0], ref["lse"], lbd, f"{c.name} splits {sp} lse")


def _long_reference(q, k, v, scale, chunk=2 ** 20):
    """attn_ref.reference of q [H, D] over k, v [Nk, D], two passes over key chunks in fp64 on the device."""
    q64 = q.double()
    H, D = q.shape
    Nk = k.shape[0]
    mx = torch.full((H, 1), -math.inf, dtype=torch.float64, device=dev)
    qk = torch.zeros((H, 1), dtype=torch.float64, device=dev)
    for j in range(0, Nk, chunk):
        kc = k[j:j + chunk].double()
        mx = torch.maximum(mx, (q64 @ kc.T * scale).amax(-1, keepdim=True))
        qk = torch.maximum(qk, (q64.abs() @ kc.abs().T).amax(-1, keepdim=True))
    l = torch.zeros((H, 1), dtype=torch.float64, device=dev)
    o = torch.zeros((H, D), dtype=torch.float64, device=dev)
    sig = torch.zeros((H, D), dtype=torch.float64, device=dev)
    vab = torch.zeros((1, D), dtype=torch.float64, device=dev)
    for j in range(0, Nk, chunk):
        kc, vc = k[j:j + chunk].double(), v[j:j + chunk].double()
        w = torch.exp(q64 @ kc.T * scale - mx)
        l += w.sum(-1, keepdim=True)
        o += w @ vc
        sig += w @ vc.abs()
        vab += vc.abs().sum(0, keepdim=True)
    rho = scale * (math.ceil(D / 16) + 16) * 2.0 ** -23 * qk
    return {"o": o / l, "lse": (mx + torch.log(l))[:, 0], "sigma": sig / l, "tau": vab / l, "rho": rho, "N": Nk, "D": D}


def _fp8_codes(shape, seed, chunk=2 ** 28):
    """Finite e4m3 codes of magnitude <= 8 with random signs, filled in chunks (no full-size temporary)."""
    out = torch.empty(shape, dtype=torch.uint8, device=dev)
    flat = out.view(-1)
    gen = torch.Generator(device=dev).manual_seed(seed)
    for i in range(0, flat.numel(), chunk):
        part = flat[i:i + chunk]
        torch.randint(0, 0x50, part.shape, dtype=torch.uint8, device=dev, generator=gen, out=part)
        part.bitwise_or_(torch.randint(0, 2, part.shape, dtype=torch.uint8, device=dev, generator=gen) << 7)
    return out.view(torch.float8_e4m3fn)


def _fp8_fp64(o, lse, q, kf, vf, c, lq, lk, what):
    """One batch of an fp8-K/V call against attn_fp8kv_ref: kf, vf are the code values as fp32 [1, Hkv, Nk, D]."""
    s = c.shape
    D = q.shape[-1]
    Tn = "bf16" if c.dtype == "bf16" else "half"
    scale = float(torch.tensor(R.kernel_scale(D), dtype=torch.float32) * torch.tensor(s["k_scale"], dtype=torch.float32))
    ref = S.reference(q, kf, vf, scale, s["causal"], [lq], [lk])
    xmax = F8.score_max(q, SR.expand(kf, q.shape[1] // kf.shape[1]), scale)
    within(o, s["v_scale"] * ref["o"], F8.o_bound(ref, D <= 128, Tn, s["v_scale"], xmax), what + " O")
    live = ~ref["empty"]
    within(lse[live], ref["lse"][live], F8.lse_bound(ref, D <= 128, xmax)[live], what + " lse")
    assert bool(torch.isneginf(lse[~live]).all()), what + " lse of empty rows"


def run_paged(c):
    s = c.shape
    T = TORCH[c.dtype]
    B, H, Hkv, Nq, D = s["B"], s["H"], s["Hkv"], s["Nq"], s["D"]
    P, ps, mp = s["num_pages"], s["page_size"], s["max_pages"]
    fp8 = s["kv"] == "e4m3"
    if fp8:
        kp, vp = _fp8_codes((P, ps, Hkv, D), 31), _fp8_codes((P, ps, Hkv, D), 32)
    else:
        kp, vp = randn((P, ps, Hkv, D), T, 31), randn((P, ps, Hkv, D), T, 32)
    q = randn((B, H, Nq, D), T, 33)
    first = P - B * mp                                   # the tables take the top B * mp pages
    table = (first + torch.arange(B * mp, dtype=torch.int32, device=dev)).view(B, mp)
    lq = torch.tensor(s["lq"], dtype=torch.int32, device=dev)
    lk = torch.tensor(s["lk"], dtype=torch.int32, device=dev)
    o, ob = guarded((B, H, Nq, D), T)
    lse, lb = guarded((B, H, Nq), torch.float32)
    kw = dict(causal=s["causal"], num_splits=1, seqlens_q=lq, seqlens_k=lk, k_scale=s["k_scale"],
              v_scale=s["v_scale"])
    with Run(c) as r:
        flash_attn.fmha_fwd(q, kp, vp, o, lse=lse, block_table=table, **kw)
    check_peak(c, r.peak)
    assert r.launches == 1
    guard_intact(ob, o.numel(), c.name + " O")
    guard_intact(lb, lse.numel(), c.name + " lse")
    # the same pages copied into a small pool, the table renumbered
    ks, vs = kp[first:].clone(), vp[first:].clone()
    so, sl = torch.empty_like(o), torch.empty_like(lse)
    flash_attn.fmha_fwd(q, ks, vs, so, lse=sl, block_table=table - first, **kw)
    same(o, so, c.name + " O")
    same(lse, sl, c.name + " lse")
    Nk = mp * ps
    kpad = PG.gather(ks.view(torch.uint8) if fp8 else ks, table - first, s["lk"], Nk)
    vpad = PG.gather(vs.view(torch.uint8) if fp8 else vs, table - first, s["lk"], Nk)
    if fp8:
        kpad, vpad = kpad.view(torch.float8_e4m3fn).float(), vpad.view(torch.float8_e4m3fn).float()
    for b in range(B):
        args = (o[b:b + 1], lse[b:b + 1], q[b:b + 1], kpad[b:b + 1], vpad[b:b + 1])
        if fp8:
            _fp8_fp64(*args, c, s["lq"][b], s["lk"][b], f"{c.name} batch {b}")
        else:
            _attn_fp64(*args, s["causal"], s["lq"][b], s["lk"][b], c.dtype, f"{c.name} batch {b}")


def run_varlen(c):
    s = c.shape
    H, Hkv, D, lens = s["H"], s["Hkv"], s["D"], s["lens"]
    B, total = len(lens), sum(lens)
    cu = [0]
    for n in lens:
        cu.append(cu[-1] + n)
    maxl = max(lens)
    cu_t = torch.tensor(cu, dtype=torch.int32, device=dev)
    q = randn((total, H, D), torch.float16, 41)
    k = randn((total, Hkv, D), torch.float16, 42)
    v = randn((total, Hkv, D), torch.float16, 43)
    o, ob = guarded((total, H, D), torch.float16)
    lse, lb = guarded((H, total), torch.float32)
    with Run(c) as r:
        flash_attn.fmha_varlen_fwd(q, k, v, o, cu_t, cu_t, maxl, maxl, causal=s["causal"], lse=lse)
    check_peak(c, r.peak)
    assert r.launches == 1
    guard_intact(ob, o.numel(), c.name + " O")
    guard_intact(lb, lse.numel(), c.name + " lse")
    cross_row = L.TWO31 // (H * D)
    seqs = sorted({0, next(b for b in range(B) if cu[b + 1] > cross_row), B - 2, B - 1})
    for b in seqs:
        n = lens[b]
        pad = lambda x: x[cu[b]:cu[b] + n].transpose(0, 1)[None].contiguous()   # noqa: E731
        qp, kp, vp = pad(q), pad(k), pad(v)
        po, pl = torch.empty_like(qp), torch.empty((1, H, n), dtype=torch.float32, device=dev)
        ln = torch.tensor([n], dtype=torch.int32, device=dev)
        flash_attn.fmha_fwd(qp, kp, vp, po, lse=pl, causal=s["causal"], num_splits=1, seqlens_q=ln, seqlens_k=ln)
        got_o = o[cu[b]:cu[b] + n].transpose(0, 1)[None]
        got_l = lse[:, cu[b]:cu[b] + n][None]
        same(got_o, po, f"{c.name} sequence {b}")
        same(got_l, pl, f"{c.name} sequence {b} lse")
        _attn_fp64(got_o, got_l, qp, kp, vp, s["causal"], n, n, "f16", f"{c.name} sequence {b}")


def run_varlen_paged(c):
    """fmha_varlen_fwd(block_table=) over the top pages of a > 2^31-element pool: bit for bit the same call on those
    pages copied into a small pool (table renumbered) and the paged seqlens call on padded Q; fp64 on every sequence."""
    s = c.shape
    B, H, Hkv, D = s["B"], s["H"], s["Hkv"], s["D"]
    P, ps, mp = s["num_pages"], s["page_size"], s["max_pages"]
    lq, lk = s["lq"], s["lk"]
    kp, vp = randn((P, ps, Hkv, D), torch.float16, 45), randn((P, ps, Hkv, D), torch.float16, 46)
    cu = [0]
    for n in lq:
        cu.append(cu[-1] + n)
    total, maxq = cu[-1], max(lq)
    q = randn((total, H, D), torch.float16, 47)
    first = P - B * mp
    table = (first + torch.arange(B * mp, dtype=torch.int32, device=dev)).view(B, mp)
    cu_t = torch.tensor(cu, dtype=torch.int32, device=dev)
    lk_t = torch.tensor(lk, dtype=torch.int32, device=dev)
    o, ob = guarded((total, H, D), torch.float16)
    lse, lb = guarded((H, total), torch.float32)

    def call(kp_, vp_, table_, o_, lse_):
        flash_attn.fmha_varlen_fwd(q, kp_, vp_, o_, cu_t, None, maxq, 0, causal=s["causal"], lse=lse_,
                                   block_table=table_, seqused_k=lk_t)
    with Run(c) as r:
        call(kp, vp, table, o, lse)
    check_peak(c, r.peak)
    assert r.launches == 1
    guard_intact(ob, o.numel(), c.name + " O")
    guard_intact(lb, lse.numel(), c.name + " lse")
    ks, vs = kp[first:].clone(), vp[first:].clone()
    so, sl = torch.empty_like(o), torch.empty_like(lse)
    call(ks, vs, table - first, so, sl)
    same(o, so, c.name + " O against the small pool")
    same(lse, sl, c.name + " lse against the small pool")
    # padded Q [B, H, maxq, D] through the paged seqlens call
    qp = torch.zeros((B, H, maxq, D), dtype=torch.float16, device=dev)
    for b in range(B):
        qp[b, :, :lq[b]] = q[cu[b]:cu[b + 1]].transpose(0, 1)
    po, pl = torch.empty_like(qp), torch.empty((B, H, maxq), dtype=torch.float32, device=dev)
    flash_attn.fmha_fwd(qp, ks, vs, po, lse=pl, causal=s["causal"], num_splits=1, block_table=table - first,
                        seqlens_q=torch.tensor(lq, dtype=torch.int32, device=dev), seqlens_k=lk_t)
    kpad = PG.gather(ks, table - first, lk, mp * ps)
    vpad = PG.gather(vs, table - first, lk, mp * ps)
    for b in range(B):
        got_o = o[cu[b]:cu[b + 1]].transpose(0, 1)[None]
        got_l = lse[:, cu[b]:cu[b + 1]][None]
        same(got_o, po[b:b + 1, :, :lq[b]], f"{c.name} sequence {b} against the padded paged call")
        same(got_l, pl[b:b + 1, :, :lq[b]], f"{c.name} sequence {b} lse against the padded paged call")
        _attn_fp64(got_o, got_l, qp[b:b + 1, :, :lq[b]], kpad[b:b + 1], vpad[b:b + 1], s["causal"], lq[b], lk[b],
                   "f16", f"{c.name} sequence {b}")


def run_edge(c):
    s = c.shape
    kind = s["kind"]
    T = TORCH[c.dtype]
    B, H, Hkv, N, D = s["B"], s["H"], s["Hkv"], s["Nq"], s["D"]
    if kind == "varlen":
        cu = torch.arange(0, (B + 1) * N, N, dtype=torch.int32, device=dev)
        total = int(cu[-1])
        q, k, v = randn((total, H, D), T, 51), randn((total, Hkv, D), T, 52), randn((total, Hkv, D), T, 53)
        o, ob = guarded((total, H, D), T)
        lse, lb = guarded((H, total), torch.float32)
        call = lambda q, k, v, o, lse, cu: flash_attn.fmha_varlen_fwd(q, k, v, o, cu, cu, N, N, causal=True, lse=lse)  # noqa
        with Run(c) as r:
            call(q, k, v, o, lse, cu)
        check_peak(c, r.peak)
        assert r.launches == 1
        guard_intact(ob, o.numel(), c.name)
        guard_intact(lb, lse.numel(), c.name + " lse")
        for b in (0, B - 1):
            a, e = int(cu[b]), int(cu[b + 1])
            so, sl = torch.empty_like(o[a:e]), torch.empty((H, e - a), dtype=torch.float32, device=dev)
            call(q[a:e], k[a:e], v[a:e], so, sl, torch.tensor([0, e - a], dtype=torch.int32, device=dev))
            same(o[a:e], so, f"{c.name} sequence {b}")
            same(lse[:, a:e], sl, f"{c.name} sequence {b} lse")
            _attn_fp64(o[a:e].transpose(0, 1)[None], lse[:, a:e][None], q[a:e].transpose(0, 1)[None],
                       k[a:e].transpose(0, 1)[None], v[a:e].transpose(0, 1)[None], True, e - a, e - a, c.dtype,
                       f"{c.name} sequence {b}")
        return
    q = randn((B, H, N, D), T, 54)
    o, ob = guarded((B, H, N, D), T)
    lse, lb = guarded((B, H, N), torch.float32)
    lq, lk = S.clamp([1 + b % N for b in range(B)], N), S.clamp([N - b % 5 for b in range(B)], N)
    lq[-1] = lk[-1] = N
    lqt, lkt = (torch.tensor(x, dtype=torch.int32, device=dev) for x in (lq, lk))
    if kind == "paged":
        kp, vp = randn((B, N, Hkv, D), T, 55), randn((B, N, Hkv, D), T, 56)    # one page of N keys per sequence
        table = torch.arange(B - 1, -1, -1, dtype=torch.int32, device=dev).view(B, 1)

        def call(sl, o, lse):
            pages = table[sl]
            flash_attn.fmha_fwd(q[sl], kp, vp, o, lse=lse, causal=True, block_table=pages, seqlens_q=lqt[sl],
                                seqlens_k=lkt[sl])
        kd = vd = None
    else:
        kd, vd = randn((B, Hkv, N, D), T, 55), randn((B, Hkv, N, D), T, 56)

        def call(sl, o, lse):
            if kind == "seqlens":
                flash_attn.fmha_fwd(q[sl], kd[sl], vd[sl], o, lse=lse, causal=True, seqlens_q=lqt[sl],
                                    seqlens_k=lkt[sl])
            else:
                flash_attn.fmha_fwd(q[sl], kd[sl], vd[sl], o, lse=lse)
    with Run(c) as r:
        call(slice(0, B), o, lse)
    check_peak(c, r.peak)
    assert r.launches == 1
    guard_intact(ob, o.numel(), c.name)
    guard_intact(lb, lse.numel(), c.name + " lse")
    for b in (0, B - 1):
        sl_ = slice(b, b + 1)
        so, sl = torch.empty_like(o[sl_]), torch.empty_like(lse[sl_])
        call(sl_, so, sl)
        same(o[sl_], so, f"{c.name} batch {b}")
        same(lse[sl_], sl, f"{c.name} batch {b} lse")
        if kind == "paged":
            kb = kp[B - 1 - b].transpose(0, 1)[None]
            vb = vp[B - 1 - b].transpose(0, 1)[None]
        else:
            kb, vb = kd[sl_], vd[sl_]
        causal, a, e = (False, N, N) if kind == "dense" else (True, lq[b], lk[b])
        _attn_fp64(o[sl_], lse[sl_], q[sl_], kb, vb, causal, a, e, c.dtype, f"{c.name} batch {b}")


# ------------------------------------------------------------------ GEMM
def _row_slices(M, N, rows=128):
    cross = L.TWO31 // N
    return [(0, rows), (cross - rows // 2, cross + rows // 2), (M - rows, M)]


def run_hgemm(c):
    s = c.shape
    M, N, K, tn, acc = s["M"], s["N"], s["K"], s["tn"], s["acc"]
    rows = s["rows"]
    a = randn((rows or M, K), torch.float16, 61)
    b = randn((N, K) if tn else (K, N), torch.float16, 62).view(K, N)
    bl = b.view(N, K).T if tn else b                      # the logical [K, N] operand
    cm, cb = guarded((M, N), torch.float16)
    mode = "f16acc" if acc == "f16" else "f16"
    with Run(c) as r:
        if rows:
            rc = _capi.lib().b200_hgemm_f16_rows(a.data_ptr(), b.data_ptr(), cm.data_ptr(), rows, N, K,
                                                 _capi.B_ROW_MAJOR_KN, s["row0"], _capi.raw_stream(0))
            _capi.check(rc, "hgemm_rows")
        else:
            hgemm.hgemm(a, b, cm, tn=tn, acc=acc)
    check_peak(c, r.peak)
    assert r.launches == 1
    guard_intact(cb, cm.numel(), c.name)
    if rows:
        row0 = s["row0"]
        assert bool(torch.isnan(cm[:64].float()).all() and torch.isnan(cm[row0 - 64:row0].float()).all()), \
            c.name + ": rows outside the shard were written"
        slices = [(0, 128), (rows - 128, rows)]
        base = row0
    else:
        slices, base = _row_slices(M, N), 0
    for r0, r1 in slices:
        small = torch.empty((r1 - r0, N), dtype=torch.float16, device=dev)
        hgemm.hgemm(a[r0:r1], b, small, tn=tn, acc=acc)
        got = cm[base + r0:base + r1]
        same(got, small, f"{c.name} rows {base + r0}..{base + r1}")
        ref = G.reference(a[r0:r1], bl, mode)
        within(got, ref["c"], G.bound(ref), f"{c.name} rows {base + r0}..{base + r1}")


def _ternary(shape, seed):
    gen = torch.Generator(device=dev).manual_seed(seed)
    return torch.randint(-1, 2, shape, dtype=torch.float32, device=dev, generator=gen)


def run_sgemm(c):
    s = c.shape
    M, N, K, mode, tn, rnd, gen = s["M"], s["N"], s["K"], s["mode"], s["tn"], s["round"], s["gen"]
    if gen == "randn":
        a = randn((M, K), torch.float32, 71)
        b = randn((N, K) if tn else (K, N), torch.float32, 72).view(K, N)
    else:
        a, b = _ternary((M, K), 71), _ternary((K, N), 72)
        if gen == "tail":                                  # zero but for the last 64 k's
            a[:, :K - 64] = 0
            b[:K - 64] = 0
    cm, cb = guarded((M, N), torch.float32)

    def call(a_, c_):
        if mode == "3xtf32":
            sgemm.sgemm_3xtf32(a_, b, c_)
        else:
            sgemm.sgemm_tf32(a_, b, c_, tn=tn, round_inputs=rnd)
    with Run(c) as r:
        call(a, cm)
    check_peak(c, r.peak)
    assert r.launches == (2 if mode == "tf32" and not rnd else 3), r.launches
    guard_intact(cb, cm.numel(), c.name)
    bl = b.view(N, K).T if tn else b
    slices = _row_slices(M, N) if gen == "randn" else [(0, M // 2), (M // 2, M)]
    for r0, r1 in slices:
        small = torch.empty((r1 - r0, N), dtype=torch.float32, device=dev)
        call(a[r0:r1], small)
        same(cm[r0:r1], small, f"{c.name} rows {r0}..{r1}")
        if gen == "randn":
            ref = G.reference(a[r0:r1], bl, "3xtf32" if mode == "3xtf32" else ("tf32" if rnd else "tf32t"))
            within(cm[r0:r1], ref["c"], G.bound(ref), f"{c.name} rows {r0}..{r1}")
    if gen != "randn":
        # {-1, 0, 1}: exact in TF32, every partial sum below 2^24, so C is the integer product bit for bit
        want = a.double() @ b.double()
        if gen == "tail":
            assert bool((want != 0).any())
        mism = int((cm.double() != want).sum())
        assert mism == 0, f"{c.name}: {mism} of {M * N} elements differ from the exact product"


# ------------------------------------------------------------------ elementwise
def run_merge(c):
    s = c.shape
    T_, H, D = s["T"], s["H"], s["D"]
    dt = TORCH[c.dtype]
    o, ob = guarded((T_, H, D), dt)
    p = o if s["in_place"] else randn((T_, H, D), dt, 81)
    if s["in_place"]:
        p.normal_(generator=torch.Generator(device=dev).manual_seed(81))
    sfx = randn((T_, H, D), dt, 82)
    pl, sl_ = randn((H, T_), torch.float32, 83), randn((H, T_), torch.float32, 84)
    olse, olb = guarded((H, T_), torch.float32)
    cross = L.TWO31 // (H * D)
    slices = [(0, 64), (cross - 32, cross + 32), (T_ - 64, T_)]
    saved = [(p[a:e].clone(), sfx[a:e].clone(), pl[:, a:e].contiguous(), sl_[:, a:e].contiguous()) for a, e in slices]
    torch.cuda.reset_peak_memory_stats()
    with Run(c) as r:
        merge_attn_states.merge_attn_states_cuda(o, p, pl, sfx, sl_, olse)
    small_bytes = sum(sum(t.numel() * t.element_size() for t in x) for x in saved)
    check_peak(c, r.peak - small_bytes)
    assert r.launches == 1
    guard_intact(ob, o.numel(), c.name)
    guard_intact(olb, olse.numel(), c.name + " lse")
    for (a, e), (ps, ss, pls, sls) in zip(slices, saved):
        so, slo = torch.empty_like(ps), torch.empty_like(pls)
        merge_attn_states.merge_attn_states_cuda(so, ps, pls, ss, sls, slo)
        same(o[a:e], so, f"{c.name} tokens {a}..{e}")
        same(olse[:, a:e], slo, f"{c.name} tokens {a}..{e} lse")
        ref = MR.reference(ps, pls, ss, sls)
        within(o[a:e], ref["o"], MR.o_bound(ref), f"{c.name} tokens {a}..{e}")
        within(olse[:, a:e], ref["lse"], MR.lse_bound(ref), f"{c.name} tokens {a}..{e} lse")


def run_rows(c):
    s = c.shape
    rows, D = s["rows"], s["D"]
    dt = TORCH[c.dtype]
    x, xb = guarded((rows, D), dt)
    x.normal_(generator=torch.Generator(device=dev).manual_seed(91))
    y, yb = (x, xb) if s["in_place"] else guarded((rows, D), dt)
    cross = L.TWO31 // D
    slices = [(0, 64), (cross - 32, min(cross + 32, rows)), (rows - 64, rows)]
    saved = [x[a:e].clone() for a, e in slices]
    small_bytes = sum(t.numel() * t.element_size() for t in saved)
    entry = c.entry

    def call(x_, y_):
        if entry == "rope_f32":
            rope.rope_f32(x_, y_)
        elif entry == "tf32_round":
            sgemm.tf32_round_(x_)
        else:
            rms_norm.rms_norm(x_, y_, 1.25)
    torch.cuda.reset_peak_memory_stats()
    with Run(c) as r:
        call(x, y)
    check_peak(c, r.peak - small_bytes)
    assert r.launches == 1
    guard_intact(yb, y.numel(), c.name)
    for (a, e), xs in zip(slices, saved):
        got = y[a:e]
        what = f"{c.name} rows {a}..{e}"
        if entry == "rope_f32":      # the position is the row: a slice would restart it, so the fp64 bound only
            want, bnd = RR.rope_reference(xs, torch.arange(a, e, device=dev))
            within(got, want, bnd, what)
            continue
        small = xs.clone() if entry == "tf32_round" else torch.empty_like(xs)
        call(xs.clone() if entry != "tf32_round" else small, small)
        same(got, small, what)
        if entry == "tf32_round":
            same(got, G.tf32(xs), what + " against tf32()")
        else:
            want, bnd = RR.rms_reference(xs, 1.25)
            within(got, want, bnd, what)


def run_rope_qk(c):
    s = c.shape
    B, H, N, D = s["B"], s["H"], s["N"], s["D"]
    q, qb = guarded((B, H, N, D), torch.float16)
    k, kb = guarded((B, H, N, D), torch.float16)
    gen = torch.Generator(device=dev).manual_seed(95)
    q.normal_(generator=gen)
    k.normal_(generator=gen)
    heads = [(0, 1), (H - 1, H)]                  # head H - 1 straddles 2^31 elements
    saved = [(q[:, a:e].clone(), k[:, a:e].clone()) for a, e in heads]
    small_bytes = sum(t.numel() * 2 for x in saved for t in x)
    torch.cuda.reset_peak_memory_stats()
    with Run(c) as r:
        fused_ops.rope_qk(q, k)
    check_peak(c, r.peak - small_bytes)
    assert r.launches == 1
    guard_intact(qb, q.numel(), c.name + " Q")
    guard_intact(kb, k.numel(), c.name + " K")
    for (a, e), (qs, ks) in zip(heads, saved):
        q0, k0 = qs.clone(), ks.clone()
        fused_ops.rope_qk(qs, ks)
        same(q[:, a:e], qs, f"{c.name} Q heads {a}..{e}")
        same(k[:, a:e], ks, f"{c.name} K heads {a}..{e}")
        for got, x0 in ((q[0, a], q0[0, 0]), (k[0, a], k0[0, 0])):
            t = torch.arange(N - 256, N, device=dev)
            want, bnd = RR.rope_reference(x0[t], t, f16_out=True)
            within(got[t], want, bnd, f"{c.name} head {a} positions {N - 256}..{N}")


RUNNERS = {
    "dense": run_dense, "seqlens": run_dense, "long_context": run_long, "paged": run_paged, "fp8": run_paged,
    "varlen": run_varlen, "rms_attn": run_rms, "grid_edge": run_edge, "hgemm": run_hgemm, "sgemm": run_sgemm,
}


def _runner(c):
    if c.entry == "fmha_f16_varlen_paged":
        return run_varlen_paged
    if c.entry == "fmha_f16_fp8kv_seqlens":
        return run_dense
    if c.family != "elementwise":
        return RUNNERS[c.family]
    if c.entry.startswith("merge"):
        return run_merge
    return run_rope_qk if c.entry == "rope_qk" else run_rows


@pytest.mark.gpu
@pytest.mark.parametrize("name", [c.name for c in L.CASES])
def test_large(name, built_lib):
    c = L.by_name()[name]
    gc.collect()
    torch.cuda.empty_cache()
    free, _ = torch.cuda.mem_get_info()
    if free < c.total + MARGIN:
        pytest.skip(f"{name}: {free / L.GiB:.2f} GiB free, the case needs {c.total / L.GiB:.2f} GiB restated "
                    f"+ {MARGIN / L.GiB:.0f} GiB margin")
    torch.cuda.reset_peak_memory_stats()
    _BASE[0] = torch.cuda.memory_allocated()
    assert _BASE[0] < BASE_LIMIT, f"{_BASE[0]} bytes still allocated before {name}"
    try:
        _runner(c)(c)
    finally:
        gc.collect()
        torch.cuda.empty_cache()
