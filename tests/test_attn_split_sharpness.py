"""The bound of a split-KV combined row (attn_split_ref.combine_bound) holds for the kernel's split + combine arithmetic
with grouped heads, and catches the mistakes GQA packing and split-KV tend to make.  CPU only (numpy).

For every kernel family each mutation of the fp64 restatement must break the bound on at least one generator
(attn_ref's and the two diagonal probes); the restatement of the kernel's arithmetic (fp32 parts with the polynomial
keys, the combine's expf / fmaf / reciprocal, one fp16 rounding) must stay inside it on all of them.
"""
import numpy as np
import pytest

import attn_mask_ref as M
import attn_ref as R
import attn_split_ref as SR
from test_attn_bound_sharpness import _poly_mask

FAMILIES = {"D<=64": 64, "64<D<=128": 128, "D>128": 136}
H, HKV = 4, 2
# (Nq, Nk, causal, splits): decode, a packed tile that straddles query heads, Nq > Nk with empty rows and splits
SHAPES = [(1, 777, False, 3), (3, 300, True, 2), (65, 200, True, 3), (150, 100, True, 4), (5, 129, False, 7)]
MUTATIONS = {
    "kv_head_h_mod_hkv": dict(head_mod=True),
    "position_r_not_r_mod_nq": dict(packed_pos=False),
    "boundary_drops_a_block": dict(boundary=-1),
    "boundary_repeats_a_block": dict(boundary=1),
    "empty_split_finite_lse": dict(empty_finite=True),
    "weights_not_renormalised": dict(renormalise=False),
}


def _cases(D, Nq, Nk):
    kbn, _ = M.kernel_shape(D)
    gens = [(g, s) for g, s in R.VARIANTS if R.usable(g, D)] + [(p, None) for p in M.PROBES]
    for i, (gen, scale) in enumerate(gens):
        q, k, v, _ = M.make_inputs(gen, 1, HKV, Nq, Nk, D, kbn, scale, seed=500 + i)
        if gen == "one_hot" or gen in M.PROBES:
            q = np.repeat(q, H // HKV, axis=1)
        else:
            q = M.make_inputs(gen, 1, H, Nq, Nk, D, kbn, scale, seed=900 + i)[0]
        yield gen, scale, q, k, v


def _truth(gen, scale, q, k, v, causal, splits):
    D = q.shape[-1]
    parts = SR.part_references(q, k, v, R.kernel_scale(D, scale), causal, splits, M.exact_scores(gen))
    full = M.reference(q, SR.expand(k, H // HKV), SR.expand(v, H // HKV), R.kernel_scale(D, scale), causal,
                       exact_scores=M.exact_scores(gen))
    want, wl, empty, ob, lb = SR.combine_bound(parts, poly=D <= 128)
    # the combination of the parts is the unsplit attention
    ne = ~empty
    assert np.array_equal(empty, full["empty"])
    assert np.allclose(want[ne], full["o"][ne], rtol=1e-9, atol=1e-12)
    return full["o"][0], full["lse"][0], empty[0], ob[0], lb[0]


def _violates(o, lse, want, wl, empty, ob, lb):
    if np.any(np.isnan(o)) or np.any(np.isnan(lse)):
        return True
    if np.any(o[empty] != 0) or np.any(lse[empty] != -np.inf):
        return True
    ne = ~empty
    return bool(np.any(np.abs(o[ne] - want[ne]) > ob[ne]) or np.any(np.abs(lse[ne] - wl[ne]) > lb[ne]))


@pytest.mark.parametrize("fam", list(FAMILIES))
def test_kernel_arithmetic_stays_inside_the_bound(fam):
    D = FAMILIES[fam]
    worst = 0.0
    for Nq, Nk, causal, splits in SHAPES:
        for gen, scale, q, k, v in _cases(D, Nq, Nk):
            want, wl, empty, ob, lb = _truth(gen, scale, q, k, v, causal, splits)
            o, lse = SR.online_split(q[0], k[0], v[0], R.kernel_scale(D, scale), causal, splits, kernel=True,
                                     poly_mask=_poly_mask(D))
            o, lse = o.astype(np.float64), lse.astype(np.float64)
            assert not _violates(o, lse, want, wl, empty, ob, lb), (gen, scale, Nq, Nk, causal, splits)
            ne = ~empty
            worst = max(worst, (np.abs(o[ne] - want[ne]) / ob[ne]).max())
    assert worst > 0.02, "the bound is far looser than the arithmetic it covers"


def test_empty_rows_and_splits_are_exact():
    """Nq > Nk, causal, more splits than blocks: rows without a key are O = 0, lse = -inf; the others are finite."""
    D, Nq, Nk = 128, 300, 129
    q, k, v, _ = M.make_inputs("randn", 1, HKV, Nq, Nk, D, 64, None, seed=5)
    q = np.repeat(q, H // HKV, axis=1)
    o, lse = SR.online_split(q[0], k[0], v[0], R.kernel_scale(D), True, 7, kernel=True, poly_mask=_poly_mask(D))
    assert np.all(o[:, :Nq - Nk] == 0) and np.all(lse[:, :Nq - Nk] == -np.inf)
    assert np.all(np.isfinite(lse[:, Nq - Nk:])) and np.all(np.isfinite(o[:, Nq - Nk:].astype(np.float32)))


@pytest.mark.parametrize("mutation", list(MUTATIONS))
@pytest.mark.parametrize("fam", list(FAMILIES))
def test_mutation_is_rejected(fam, mutation):
    D = FAMILIES[fam]
    caught = []
    for Nq, Nk, causal, splits in SHAPES:
        for gen, scale, q, k, v in _cases(D, Nq, Nk):
            want, wl, empty, ob, lb = _truth(gen, scale, q, k, v, causal, splits)
            o, lse = SR.online_split(q[0], k[0], v[0], R.kernel_scale(D, scale), causal, splits, **MUTATIONS[mutation])
            if _violates(o, lse, want, wl, empty, ob, lb):
                caught.append(f"{gen}@{scale} ({Nq},{Nk},{causal},{splits})")
    assert caught, f"no generator catches {mutation} in family {fam}"
    print(f"{fam}: {mutation} rejected by {', '.join(caught[:6])}{' ...' if len(caught) > 6 else ''}")
