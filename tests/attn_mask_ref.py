"""fp64 reference of masked attention (separate query / key lengths, causal), the probes that pin the diagonal, and a
CPU restatement of the kernel's masked online softmax.  Used by test_attn_causal_gpu.py and test_attn_causal_sharpness.py.

Semantics (csrc/attn_sm90.cuh): q [.., Nq, D], k and v [.., Nk, D]; causal masks key j for query i when j > i + diag,
diag = Nk - Nq (bottom-right alignment).  Rows with i + diag < 0 see no key: O = 0 and lse = -inf.

The bound is attn_ref.o_bound / lse_bound unchanged, evaluated on the masked reference:
  * every sum over keys runs over the visible keys only (sigma, tau, the score-error term rho), and N = Nk stays in the
    fp32 summation terms, which is conservative since a row adds at most Nk keys;
  * a masked key adds exactly 0 to P V (its P is 0 in fp16) and at most 2^-126 (exp2_fma_pipe(-inf)) to l, far below
    the 2^-23 terms of the bound.
Empty rows carry sigma = tau = 0, so their O bound is 2^-24; the tests demand O == 0 and lse == -inf there exactly.
"""
from __future__ import annotations

import math

import numpy as np
import torch

import attn_ref as R

LOG2E = R.LOG2E


def visible(Nq, Nk, causal, xp=np, device=None, diag_shift=0, top_left=False):
    """[Nq, Nk] bool: key j visible to query i.  diag_shift / top_left restate mistakes for the sharpness test."""
    diag = (0 if top_left else Nk - Nq) + diag_shift
    if xp is torch:
        i = torch.arange(Nq, device=device)[:, None]
        j = torch.arange(Nk, device=device)[None, :]
        return (j <= i + diag) if causal else torch.ones(Nq, Nk, dtype=torch.bool, device=device)
    i, j = np.arange(Nq)[:, None], np.arange(Nk)[None, :]
    return (j <= i + diag) if causal else np.ones((Nq, Nk), bool)


def empty_rows(Nq, Nk, causal):
    """[Nq] bool: rows without a visible key."""
    return np.arange(Nq) + (Nk - Nq) < 0 if causal else np.zeros(Nq, bool)


def reference(q, k, v, scale, causal, exact_scores=False):
    """Masked fp64 attention of [..., Nq, D] / [..., Nk, D] inputs (numpy or torch): the dict of attn_ref.reference."""
    is_t = isinstance(q, torch.Tensor)
    xp = torch if is_t else np
    q, k, v = (x.double() if is_t else np.asarray(x, np.float64) for x in (q, k, v))
    Nq, Nk, D = q.shape[-2], k.shape[-2], q.shape[-1]
    vis = visible(Nq, Nk, causal, xp, q.device if is_t else None)
    kt = k.swapaxes(-1, -2)
    s = (q @ kt) * scale
    s = xp.where(vis, s, -math.inf)
    mx = s.amax(dim=-1, keepdim=True) if is_t else s.max(axis=-1, keepdims=True)
    empty = xp.isinf(mx)
    w = xp.exp(s - xp.where(empty, 0.0, mx))
    l = w.sum(-1, keepdims=True) if not is_t else w.sum(-1, keepdim=True)
    ls = xp.where(empty, 1.0, l)
    p = w / ls
    visf = vis.double() if is_t else vis.astype(np.float64)
    if exact_scores:
        rho = xp.zeros_like(mx)
    else:
        qk = xp.where(vis, xp.abs(q) @ xp.abs(kt), 0.0)
        rho = scale * (math.ceil(D / 16) + 16) * 2.0 ** -23 * (qk.amax(dim=-1, keepdim=True) if is_t
                                                                 else qk.max(axis=-1, keepdims=True))
    lse = xp.where(empty, -math.inf, mx + xp.log(ls))[..., 0]
    return {"o": p @ v, "lse": lse, "sigma": p @ xp.abs(v), "tau": (visf @ xp.abs(v)) / ls, "rho": rho,
            "N": Nk, "D": D, "empty": empty[..., 0]}


# ------------------------------------------------------------------ generators
PROBES = ("diag_gather", "future_max")


def make_inputs(gen, B, H, Nq, Nk, D, kbn, scale=None, seed=0):
    """Seeded fp16 q [B,H,Nq,D], k, v [B,H,Nk,D] and the row -> key map `target` of the probes (else None).

    attn_ref's generators: keys and values from attn_ref.make_inputs at Nk, queries from it at Nq (another seed; the
    query side of every generator is position-free), or its own inputs when Nq = Nk.  `one_hot` at Nq != Nk keeps the
    codes of the longer side.
    diag_gather  q_i = c code(k_{i+diag}) (attn_ref's one_hot codes, >= 48 nats of gap): O_i = V_{i+diag} exactly
                 when the diagonal is right, another row of V when it is off by one either way.
    future_max   q_i = c code(k_{i+diag+1}): the key just past the diagonal outscores every visible key by >= 48 nats,
                 so a leaked key takes over its row.  (The last row, which has no key past it, targets its diagonal.)
    """
    if gen in PROBES:
        assert D >= 32
        _, k, v, _ = R.make_inputs("one_hot", B, H, Nk, D, kbn, scale, seed)
        c = np.float16(24.0 / R.kernel_scale(D, scale))
        shift = 0 if gen == "diag_gather" else 1
        target = np.clip(np.arange(Nq) + (Nk - Nq) + shift, 0, Nk - 1)
        q = (k[:, :, target].astype(np.float32) * np.float32(c)).astype(np.float16)
        return np.ascontiguousarray(q), k, v, target
    if Nq == Nk:
        q, k, v, _ = R.make_inputs(gen, B, H, Nk, D, kbn, scale, seed)
        return q, k, v, None
    if gen == "one_hot":
        q, k, v, _ = R.make_inputs(gen, B, H, max(Nq, Nk), D, kbn, scale, seed)
        return np.ascontiguousarray(q[:, :, -Nq:]), np.ascontiguousarray(k[:, :, :Nk]), \
            np.ascontiguousarray(v[:, :, :Nk]), None
    _, k, v, _ = R.make_inputs(gen, B, H, Nk, D, kbn, scale, seed)
    q, _, _, _ = R.make_inputs(gen, B, H, Nq, D, kbn, scale, seed + 7919)
    return q, k, v, None


def exact_scores(gen):
    return gen == "one_hot" or gen in PROBES


# ------------------------------------------------------------------ CPU restatement of the kernel
def kernel_shape(D):
    """(keys per block, query rows per CTA) of the kernel fmha_dispatch picks for head dim D."""
    _, kbn = R.family(D)
    return kbn, (64 if D > 128 else 128)


def online(q, k, v, scale, D, causal, kernel=False, poly_mask=0, diag_shift=0, top_left=False, nkv_short=False,
           empty_finite=False):
    """The masked online softmax of one head ([Nq, D] / [Nk, D] numpy) the way the kernel walks it: query tiles of
    kernel_shape(D)[1] rows, each over its first nkv key blocks, the tail and diagonal masks, the m == -inf guard.

    kernel=False: float64 (the mutations apply to this form); kernel=True: the kernel's fp32 / fp16 / polynomial
    arithmetic as in attn_ref.online.  Mutations: diag_shift (+1 leaks a key, -1 drops the diagonal), top_left
    (SDPA's alignment), nkv_short (the CTA's last key block skipped), empty_finite (an empty row reported with a
    finite lse).  Returns (O, lse)."""
    kbn, rows = kernel_shape(D)
    ft = np.float32 if kernel else np.float64
    c = ft(ft(scale) * ft(LOG2E))
    Nq, Nk = q.shape[0], k.shape[0]
    diag = (0 if top_left else Nk - Nq) + diag_shift
    num_kv = -(-Nk // kbn)
    s_all = q.astype(ft) @ k.astype(ft).T
    o_out = np.zeros((Nq, v.shape[1]), np.float16 if kernel else np.float64)
    lse_out = np.zeros(Nq, ft)
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        for q0 in range(0, Nq, rows):
            n = min(rows, Nq - q0)
            if causal:
                keys = q0 + rows + diag
                nkv = 0 if keys <= 0 else min(num_kv, -(-keys // kbn))
            else:
                nkv = num_kv
            if nkv_short:
                nkv = max(0, nkv - 1)
            m = np.full((n, 1), -np.inf, ft)
            l = np.zeros((n, 1), ft)
            o = np.zeros((n, v.shape[1]), ft)
            row = np.arange(q0, q0 + n)[:, None]
            for b in range(nkv):
                b0 = b * kbn
                key = np.arange(b0, min(b0 + kbn, Nk))[None, :]
                s = s_all[q0:q0 + n, b0:b0 + kbn].copy()
                if causal:
                    s[key > row + diag] = -np.inf
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
                pv = (p.astype(np.float16).astype(ft) if kernel else p) @ v[b0:b0 + kbn].astype(ft)
                o = (o * alpha + pv).astype(ft)
            empty = m == -np.inf
            inv = np.where(empty, ft(0), ft(1) / np.where(empty, ft(1), l))
            o = (o * inv).astype(ft)
            lse = np.where(empty, -np.inf, (m + np.log2(np.where(empty, ft(1), l))) * ft(math.log(2.0)))
            if empty_finite:   # what a kernel reports that tells an empty row by l: ln(2^-126) from a polynomial key
                lse = np.where(empty, ft(-126 * math.log(2.0)), lse)
            o_out[q0:q0 + n] = o.astype(np.float16) if kernel else o
            lse_out[q0:q0 + n] = lse[:, 0]
    return o_out, lse_out
