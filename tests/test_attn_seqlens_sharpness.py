"""The per-sequence arithmetic of attn_fwd_seqlens_kernel restated on the CPU (float64, one K/V group of one sequence,
poisoned padding) meets the fp64 reference, and each restated mistake breaks that: the checks of
test_attn_seqlens_gpu.py can tell these mistakes apart from a correct kernel."""
import math

import numpy as np
import pytest

import attn_mask_ref as M
import attn_seqlens_ref as S
import attn_split_ref as SR

MISTAKES = ("diag_padded", "tail_padded", "short_block", "v_unzeroed", "pad_computed", "split_short")


def restate(q, k, v, scale, causal, lq, lk, splits=1, mistake=None):
    """q [G, Nq, D], k, v [Nk, D] (padding poisoned): (O [G, Nq, D], lse [G, Nq]) as the kernel computes them, with
    the parts of a split combined."""
    G, Nq, D = q.shape
    Nk = k.shape[0]
    kbn, _ = M.kernel_shape(D)
    mut = {"diag_padded": (Nq, Nk)} if mistake == "diag_padded" else {}
    if mistake == "short_block":
        mut["short"] = 1
    key_end = Nk if mistake == "tail_padded" else lk
    diag = Nk - Nq if mistake == "diag_padded" else lk - lq
    vz = v.copy()
    if mistake != "v_unzeroed":
        vz[lk:] = 0.0                                   # the one partial block's rows past Lk_b; later blocks unvisited
    qp = q.reshape(G * Nq, D)
    pos = np.arange(G * Nq) % Nq
    o_out = np.zeros((G * Nq, D))
    l_out = np.full(G * Nq, -math.inf)
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        for rows, nkv in S.tiles(G, Nq, D, causal, lq, lk, **mut):
            rng = SR.split_ranges(nkv, splits)
            if mistake == "split_short" and splits > 1:
                rng[-1] = (rng[-1][0], max(rng[-1][0], rng[-1][1] - 1))
            parts = []
            for b_, e_ in rng:
                s = qp[rows] @ k[b_ * kbn:e_ * kbn].T * scale
                key = np.arange(b_ * kbn, b_ * kbn + s.shape[1])[None, :]
                s = np.where(key >= key_end, -math.inf, s)
                if causal:
                    s = np.where(key > pos[rows][:, None] + diag, -math.inf, s)
                m = s.max(axis=1, keepdims=True) if s.shape[1] else np.full((len(rows), 1), -math.inf)
                mb = np.where(m == -math.inf, 0.0, m)
                p = np.exp(s - mb)
                l = p.sum(axis=1, keepdims=True)
                o = p @ vz[b_ * kbn:e_ * kbn] / np.where(m == -math.inf, 1.0, l)
                lse = np.where(m[:, 0] == -math.inf, -math.inf, (mb + np.log(l))[:, 0])
                if mistake != "pad_computed":
                    pad = pos[rows] >= lq
                    o[pad], lse[pad] = 0.0, -math.inf
                parts.append((o, lse))
            lses = np.stack([x[1] for x in parts])
            top = np.maximum(lses.max(axis=0), -np.finfo(np.float32).max)
            w = np.exp(lses - top)
            den = w.sum(axis=0)
            o_out[rows] = sum(w[z][:, None] * parts[z][0] for z in range(len(parts))) / np.maximum(den, 1.0)[:, None]
            l_out[rows] = np.log(den) + top
    return o_out.reshape(G, Nq, D), l_out.reshape(G, Nq)


def _case(G, Nq, Nk, D, lq, lk, seed):
    r = np.random.default_rng(seed)
    q, k, v = r.standard_normal((G, Nq, D)), r.standard_normal((Nk, D)), r.standard_normal((Nk, D))
    q[:, lq:], k[lk:], v[lk:] = math.nan, math.nan, math.nan
    return q, k, v


def _ok(q, k, v, causal, lq, lk, got):
    G, Nq, D = q.shape
    vis = S.visible(Nq, k.shape[0], lq, lk, causal)
    qc, kc, vc = np.nan_to_num(q), np.nan_to_num(k), np.nan_to_num(v)
    ref = SR.masked_reference(qc[None], kc[None, None], vc[None, None], 1 / math.sqrt(D), vis, True)
    o, lse = got
    if np.isnan(o).any() or np.isnan(lse).any():
        return False
    empty = ref["empty"][0]
    if not ((o[empty] == 0).all() and (lse[empty] == -math.inf).all()):
        return False
    return bool(np.allclose(o[~empty], ref["o"][0][~empty], atol=1e-9)
                and np.allclose(lse[~empty], ref["lse"][0][~empty], atol=1e-9))


# (G, Nq, Nk, D, lq, lk, causal, splits): decoding, speculative and chunked prefill over a padded cache
SHAPES = [(4, 1, 400, 128, 1, 259, False, 1), (2, 5, 400, 64, 3, 200, True, 1), (1, 130, 400, 136, 100, 330, True, 1),
          (4, 5, 700, 128, 5, 517, True, 3), (2, 130, 700, 64, 90, 600, True, 4), (8, 1, 700, 136, 1, 450, False, 5)]


@pytest.mark.parametrize("shape", SHAPES)
def test_restatement_meets_the_reference(shape):
    G, Nq, Nk, D, lq, lk, causal, splits = shape
    q, k, v = _case(G, Nq, Nk, D, lq, lk, seed=Nk + lq)
    assert _ok(q, k, v, causal, lq, lk, restate(q, k, v, 1 / math.sqrt(D), causal, lq, lk, splits))


@pytest.mark.parametrize("mistake", MISTAKES)
def test_each_mistake_is_caught(mistake):
    caught = []
    for G, Nq, Nk, D, lq, lk, causal, splits in SHAPES:
        q, k, v = _case(G, Nq, Nk, D, lq, lk, seed=Nk + lq)
        got = restate(q, k, v, 1 / math.sqrt(D), causal, lq, lk, splits, mistake)
        caught.append(not _ok(q, k, v, causal, lq, lk, got))
    assert any(caught), f"{mistake} passes every shape"
