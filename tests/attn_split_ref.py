"""Grouped-query attention and split-KV (b200_fmha_fwd_f16_gqa): the kernel's key ranges, an fp64 reference of every
split's part, the bound of a combined row, and a CPU restatement of the split + combine arithmetic on top of
attn_mask_ref.online.  Used by test_attn_gqa_gpu.py and test_attn_split_sharpness.py.

Semantics.  q [B,H,Nq,D], k and v [B,Hkv,Nk,D], G = H / Hkv: query head h reads K/V head h // G.  The kernel packs the
G query heads of a K/V head into G*Nq rows; packed row r = g*Nq + i is query head hk*G + g at position i = r % Nq, which
the causal mask uses.  A CTA owns `rows` consecutive packed rows (attn_mask_ref.kernel_shape) and visits nkv key blocks:
all of them, or with the mask those left of the diagonal of the greatest position among its rows.  With the mask and
Nq >= `rows` every query head has tiles of its own (a tile's rows past its head's end are not stored).  Split z of S runs
blocks [nkv*z // S, nkv*(z+1) // S) and writes its fp32 normalised O_z and lse_z; the combine forms
    top = max_z lse_z,   w_z = expf(lse_z - top),   O = fp16(sum_z w_z O_z * (1 / sum_z w_z)),   lse = logf(sum_z w_z) + top.

Bound of a combined row (`combine_bound`).  The parts are exact attention over disjoint key sets, so with the fp64 part
results (O*_z, L*_z) and W_z = exp(L*_z - L*) (L* = logsumexp of the L*_z, the full lse) the truth is O* = sum_z W_z O*_z.
What the combine receives and does, term by term:
  1. Part errors.  O_z is the kernel's fp32 O of the part, never rounded to fp16: |O_z - O*_z| <= pre_z, attn_ref.o_bound's
     bound before the final rounding, evaluated on the part's masked reference.
  2. Weight errors.  The weight of part z is perturbed by a relative factor exp(eps_z) / sum_t W_t exp(eps_t) with
     |eps_z| <= a_z := e_z + d_z: e_z is the part's lse bound (attn_ref.lse_bound on the part) and d_z the error of the
     computed expf(lse_z - top): 2 ulp of expf (CUDA guide) <= 2^-22, plus the fp32 rounding of the argument,
     2^-24 (Delta_z + 2 A + 1) with Delta_z = max_t L*_t - L*_z and A = max_z a_z.  So each weight moves by at most
     W_z (a_z + A) exp(a_z + A) relative, and since the perturbed weights still sum to 1,
        sum_z (w'_z - W_z) O*_z = sum_z (w'_z - W_z)(O*_z - O*):   |.| <= sum_z W_z (a_z + A) exp(a_z + A) |O*_z - O*|.
     The part errors go through the perturbed weights: sum_z W_z exp(a_z + A) pre_z.
  3. The combine's fp32 arithmetic: S - 1 additions of the divisor, S fused multiply-adds per element, one reciprocal and
     one multiply, each rounding once (2^-24 relative of a value at most sum_z w_z |O_z|):
        (3 S + 2) 2^-24 sum_z W_z exp(a_z + A) (|O*_z| + pre_z).
  4. One rounding to fp16: U16 (|O*| + terms 1..3) + 2^-24 (the subnormal spacing covers the half-ulp there).
For S = 2 this is test_chunked_prefill_composes_with_merge's bound with the fp32 terms made explicit.  lse: the weighted
part lse errors and expf errors (at most A), the divisor's additions ((S - 1) 2^-24), logf (1 ulp of ln(sum w) <= ln S,
<= 2^-22 (ln S + 1)) and the final addition (2^-24 |L*|), plus 2^-24 for lse_z's own fp32 rounding already inside A.
Empty parts (no visible key in the range) carry weight 0 exactly (lse -inf); a row all of whose parts are empty must be
O = 0 and lse = -inf exactly.  Nothing here is fitted to measurements.
"""
from __future__ import annotations

import math

import numpy as np
import torch

import attn_mask_ref as M
import attn_ref as R

LOG2E = R.LOG2E
FLT_MAX = float(np.finfo(np.float32).max)


# ------------------------------------------------------------------ the kernel's key ranges
def tile_blocks(q0, rows_per_cta, rows, Nq, Nk, kbn, causal, packed_pos=True):
    """Key blocks a CTA whose packed rows start at q0 visits (csrc/attn_sm90.cuh kv_blocks).  packed_pos=False restates
    the mistake of taking the packed row for the position."""
    num_kv = -(-Nk // kbn)
    if not causal:
        return num_kv
    last = min(q0 + rows_per_cta, rows) - 1
    if packed_pos:
        rows_end = Nq if last // Nq != q0 // Nq else last % Nq + 1
    else:
        rows_end = last + 1
    keys = rows_end + Nk - Nq
    return 0 if keys <= 0 else min(num_kv, -(-keys // kbn))


def tiles(G, Nq, Nk, D, causal, packed_pos=True):
    """[(packed rows stored by the CTA, its nkv)] over the G*Nq packed rows of a K/V head (csrc/attn_sm90.cuh)."""
    kbn, per = M.kernel_shape(D)
    rows = G * Nq
    if causal and Nq >= per and packed_pos:
        out = []
        for g in range(G):
            for t0 in range(0, Nq, per):
                r = np.arange(g * Nq + t0, g * Nq + min(t0 + per, Nq))
                out.append((r, tile_blocks(t0, per, Nq, Nq, Nk, kbn, causal)))
        return out
    return [(np.arange(q0, min(q0 + per, rows)), tile_blocks(q0, per, rows, Nq, Nk, kbn, causal, packed_pos))
            for q0 in range(0, rows, per)]


def split_ranges(nkv, splits):
    return [(nkv * z // splits, nkv * (z + 1) // splits) for z in range(splits)]


def part_masks(G, Nq, Nk, D, causal, splits):
    """[S, G*Nq, Nk] bool: key j is in split z of packed row r and visible to it."""
    kbn, _ = M.kernel_shape(D)
    out = np.zeros((splits, G * Nq, Nk), bool)
    vis = M.visible(Nq, Nk, causal)
    for r, nkv in tiles(G, Nq, Nk, D, causal):
        for z, (b, e) in enumerate(split_ranges(nkv, splits)):
            out[z, r, b * kbn:min(e * kbn, Nk)] = True
    return out & np.tile(vis, (G, 1))[None]


# ------------------------------------------------------------------ fp64 references
def expand(k, G):
    """K/V heads repeated for their G query heads: [B,Hkv,..] -> [B,Hkv*G,..] (torch.repeat_interleave semantics)."""
    if isinstance(k, torch.Tensor):
        return k.repeat_interleave(G, dim=1)
    return np.repeat(k, G, axis=1)


def masked_reference(q, k, v, scale, vis, exact_scores=False):
    """attn_mask_ref.reference with an arbitrary visibility mask vis [..., Nq, Nk] (bool, broadcast over q's batch)."""
    is_t = isinstance(q, torch.Tensor)
    xp = torch if is_t else np
    q, k, v = (x.double() if is_t else np.asarray(x, np.float64) for x in (q, k, v))
    D = q.shape[-1]
    kt = k.swapaxes(-1, -2)
    s = xp.where(vis, (q @ kt) * scale, -math.inf)
    mx = s.amax(dim=-1, keepdim=True) if is_t else s.max(axis=-1, keepdims=True)
    empty = xp.isinf(mx)
    w = xp.exp(s - xp.where(empty, 0.0, mx))
    l = w.sum(-1, keepdim=True) if is_t else w.sum(-1, keepdims=True)
    ls = xp.where(empty, 1.0, l)
    p = w / ls
    visf = vis.expand(s.shape).double() if is_t else np.broadcast_to(vis, s.shape).astype(np.float64)
    if exact_scores:
        rho = xp.zeros_like(mx)
    else:
        qk = xp.where(vis, xp.abs(q) @ xp.abs(kt), 0.0)
        rho = scale * (math.ceil(D / 16) + 16) * 2.0 ** -23 * (qk.amax(dim=-1, keepdim=True) if is_t
                                                                 else qk.max(axis=-1, keepdims=True))
    lse = xp.where(empty, -math.inf, mx + xp.log(ls))[..., 0]
    return {"o": p @ v, "lse": lse, "sigma": p @ xp.abs(v), "tau": (visf @ xp.abs(v)) / ls, "rho": rho,
            "N": k.shape[-2], "D": D, "empty": empty[..., 0]}


def head_masks(masks, H, G, Nq):
    """[S, G*Nq, Nk] packed-row masks -> [S, H, Nq, Nk]: query head h uses the rows of its index within its group."""
    S, _, Nk = masks.shape
    m = masks.reshape(S, G, Nq, Nk)
    return m[:, np.arange(H) % G]


def part_references(q, k, v, scale, causal, splits, exact_scores=False):
    """fp64 references of the S parts of every row: list of dicts as attn_mask_ref.reference returns (q [B,H,Nq,D],
    k, v [B,Hkv,Nk,D]; numpy or torch)."""
    B, H, Nq, D = q.shape
    G = H // k.shape[1]
    Nk = k.shape[2]
    ke, ve = expand(k, G), expand(v, G)
    masks = head_masks(part_masks(G, Nq, Nk, D, causal, splits), H, G, Nq)
    if isinstance(q, torch.Tensor):
        masks = torch.from_numpy(masks).to(q.device)
    return [masked_reference(q, ke, ve, scale, masks[z][None], exact_scores) for z in range(splits)]


def combine_bound(parts, poly):
    """(O*, L*, empty, O bound, lse bound) of the combined rows from the parts' fp64 references (see the docstring)."""
    is_t = isinstance(parts[0]["o"], torch.Tensor)
    xp = torch if is_t else np
    S = len(parts)
    lse = xp.stack([p["lse"] for p in parts])                          # [S, ...rows]
    top = lse.amax(0) if is_t else lse.max(axis=0)
    empty = xp.isinf(top)
    topf = xp.where(empty, 0.0, top)
    W = xp.exp(lse - topf)
    W = W / xp.where(empty, 1.0, W.sum(0))                              # W_z, 0 for empty parts
    L = xp.where(empty, -math.inf, topf + xp.log(xp.where(empty, 1.0, xp.exp(lse - topf).sum(0))))
    pe = [p["empty"] for p in parts]
    e = xp.stack([xp.where(pe[z], 0.0, R.lse_bound(parts[z], poly)) for z in range(S)])
    delta = xp.where(xp.stack(pe), 0.0, topf - lse)
    a0 = e + 2.0 ** -22 + 2.0 ** -24
    A0 = a0.amax(0) if is_t else a0.max(axis=0)
    a = a0 + 2.0 ** -24 * (delta + 2 * A0)
    A = a.amax(0) if is_t else a.max(axis=0)
    o = sum(W[z][..., None] * parts[z]["o"] for z in range(S))
    term1 = term2 = term3 = 0.0
    for z in range(S):
        pre = xp.where(pe[z][..., None], 0.0, R.o_bound(parts[z], poly)[0])
        g = (W[z] * xp.exp(a[z] + A))[..., None]
        term1 = term1 + g * pre
        term2 = term2 + g * (a[z] + A)[..., None] * abs(parts[z]["o"] - o)
        term3 = term3 + g * (abs(parts[z]["o"]) + pre)
    pre_all = term1 + term2 + (3 * S + 2) * 2.0 ** -24 * term3
    ob = pre_all + R.U16 * (abs(o) + pre_all) + 2.0 ** -24
    lb = A + (S + 1) * 2.0 ** -24 + 2.0 ** -22 * (math.log(S) + 1) + 2.0 ** -24 * abs(xp.where(empty, 0.0, L))
    return o, L, empty, ob, lb


# ------------------------------------------------------------------ CPU restatement of split + combine
def online_split(q, k, v, scale, causal, splits, kernel=False, poly_mask=0, head_mod=False, packed_pos=True,
                 boundary=0, empty_finite=False, renormalise=True):
    """The kernel's split-KV GQA of one batch: q [H, Nq, D], k, v [Hkv, Nk, D] numpy.  Returns (O [H,Nq,D], lse [H,Nq]).

    kernel=False: float64 (the mutations apply to this form); kernel=True: fp32 parts with attn_mask_ref.online's
    arithmetic and the combine in fp32 (expf, fmaf order, reciprocal, one fp16 rounding).  Mutations: head_mod (query
    head h reads K/V head h % Hkv), packed_pos=False (the mask takes the packed row r as position), boundary = -1 / +1
    (the first split boundary drops / repeats one key block), empty_finite (an empty split reports a finite lse),
    renormalise=False (the combined O is not divided by the sum of the weights)."""
    H, Nq, D = q.shape
    Hkv, Nk = k.shape[0], k.shape[1]
    G = H // Hkv
    kbn, per = M.kernel_shape(D)
    ft = np.float32 if kernel else np.float64
    c = ft(ft(scale) * ft(LOG2E))
    num_kv = -(-Nk // kbn)
    groups = [([h], h % Hkv) for h in range(H)] if head_mod else [(list(range(hk * G, hk * G + G)), hk)
                                                                    for hk in range(Hkv)]
    o_out = np.zeros((H, Nq, v.shape[-1]), np.float16 if kernel else np.float64)
    l_out = np.zeros((H, Nq), ft)
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        for heads, hk in groups:
            g = len(heads)
            rows = g * Nq
            qp = q[heads].reshape(rows, D)
            s_all = qp.astype(ft) @ k[hk].astype(ft).T
            pos = np.arange(rows) % Nq if packed_pos else np.arange(rows)
            po = np.zeros((splits, rows, v.shape[-1]), ft)
            pl = np.full((splits, rows), -np.inf, ft)
            for rr, nkv in tiles(g, Nq, Nk, D, causal, packed_pos):
                q0, n = rr[0], len(rr)
                rng = split_ranges(nkv, splits)
                if boundary and splits > 1 and rng[0][1] > rng[0][0]:
                    rng[0] = (rng[0][0], min(num_kv, rng[0][1] + boundary))
                for z, (b_, e_) in enumerate(rng):
                    m = np.full((n, 1), -np.inf, ft)
                    l = np.zeros((n, 1), ft)
                    o = np.zeros((n, v.shape[-1]), ft)
                    row = pos[q0:q0 + n][:, None]
                    for b in range(b_, e_):
                        b0 = b * kbn
                        key = np.arange(b0, min(b0 + kbn, Nk))[None, :]
                        s = s_all[q0:q0 + n, b0:b0 + kbn].copy()
                        if causal:
                            s[key > row + (Nk - Nq)] = -np.inf
                        mn = np.maximum(m, (s.max(axis=1, keepdims=True) * c).astype(ft))
                        mb = np.where(mn == -np.inf, ft(0), mn)
                        alpha = np.exp2(m - mb).astype(ft)
                        x = (s.astype(np.float64) * np.float64(c) - mb).astype(ft)
                        p = np.exp2(x).astype(ft)
                        if kernel and poly_mask:
                            pair = (key[0] % 32) // 2
                            sel = ((poly_mask >> pair) & 1).astype(bool)
                            p[:, sel] = R.exp2_fma_pipe(x[:, sel])
                        m = mn
                        l = (l * alpha + p.sum(axis=1, keepdims=True)).astype(ft)
                        pv = (p.astype(np.float16).astype(ft) if kernel else p) @ v[hk, b0:b0 + kbn].astype(ft)
                        o = (o * alpha + pv).astype(ft)
                    emp = m == -np.inf
                    inv = np.where(emp, ft(0), ft(1) / np.where(emp, ft(1), l))
                    po[z, q0:q0 + n] = (o * inv).astype(ft)
                    lz = np.where(emp, -np.inf, (m + np.log2(np.where(emp, ft(1), l))) * ft(math.log(2.0)))
                    if empty_finite:
                        lz = np.where(emp, ft(-126 * math.log(2.0)), lz)
                    pl[z, q0:q0 + n] = lz[:, 0]
            top = np.maximum(pl.max(axis=0), ft(-FLT_MAX))
            acc = np.zeros((rows, v.shape[-1]), ft)
            den = np.zeros(rows, ft)
            for z in range(splits):
                w = np.exp((pl[z] - top).astype(ft)).astype(ft)
                den = (den + w).astype(ft)
                acc = (w[:, None].astype(np.float64) * po[z] + acc).astype(ft)   # fmaf: one rounding
            inv = (ft(1) / np.maximum(den, ft(1))).astype(ft) if renormalise else np.ones(rows, ft)
            res = (acc * inv[:, None]).astype(ft)
            lse = (np.log(den).astype(ft) + top).astype(ft)
            o_out[heads] = (res.astype(np.float16) if kernel else res).reshape(g, Nq, -1)
            l_out[heads] = lse.reshape(g, Nq)
    return o_out, l_out
