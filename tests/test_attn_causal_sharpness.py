"""The masked attention bound (attn_ref's bound on attn_mask_ref's masked reference) catches the mistakes a causal /
separate-length kernel tends to make, and holds for the kernel's own arithmetic with the mask.  CPU only (numpy).

For every kernel family and (Nq, Nk) below, each mutation applied to the fp64 masked online softmax must break the
bound on at least one generator (attn_ref's and the two diagonal probes); the restatement of the kernel's arithmetic
(fp32 statistics, P in fp16, the polynomial keys, the m == -inf guard, fp16 O) must stay inside it on all of them.
"""
import numpy as np
import pytest

import attn_mask_ref as M
import attn_ref as R
from test_attn_bound_sharpness import _poly_mask

# family -> head dim; shapes: equal lengths, Nq < Nk with a diagonal inside a block, Nq > Nk with empty rows
FAMILIES = {"D<=64": 64, "64<D<=128": 128, "D>128": 136}
SHAPES = [(257, 257), (129, 300), (300, 129)]
MUTATIONS = {
    "diagonal_plus_1": dict(diag_shift=1),
    "diagonal_minus_1": dict(diag_shift=-1),
    "top_left_alignment": dict(top_left=True),
    "last_block_skipped": dict(nkv_short=True),
    "empty_row_finite": dict(empty_finite=True),
}


def _cases(D, Nq, Nk):
    kbn, _ = M.kernel_shape(D)
    gens = [(g, s) for g, s in R.VARIANTS if R.usable(g, D)] + [(p, None) for p in M.PROBES]
    for i, (gen, scale) in enumerate(gens):
        q, k, v, _ = M.make_inputs(gen, 1, 1, Nq, Nk, D, kbn, scale, seed=300 + i)
        yield gen, scale, q[0, 0], k[0, 0], v[0, 0]


def _truth(gen, scale, q, k, v):
    D = q.shape[-1]
    ref = M.reference(q, k, v, R.kernel_scale(D, scale), causal=True, exact_scores=M.exact_scores(gen))
    _, bound = R.o_bound(ref, poly=D <= 128)
    return ref, bound, R.lse_bound(ref, poly=D <= 128)


def _violates(o, lse, ref, bound, lb):
    """True when O or lse leaves the bound; empty rows must be O == 0 and lse == -inf exactly."""
    e = ref["empty"]
    if np.any(o[e] != 0) or np.any(lse[e] != -np.inf):
        return True
    ne = ~e
    return bool(np.any(np.abs(o[ne] - ref["o"][ne]) > bound[ne])
                or np.any(np.abs(lse[ne] - ref["lse"][ne]) > lb[ne]))


@pytest.mark.parametrize("Nq,Nk", SHAPES)
@pytest.mark.parametrize("fam", list(FAMILIES))
def test_kernel_arithmetic_stays_inside_the_bound(fam, Nq, Nk):
    D = FAMILIES[fam]
    worst = 0.0
    for gen, scale, q, k, v in _cases(D, Nq, Nk):
        ref, bound, lb = _truth(gen, scale, q, k, v)
        o, lse = M.online(q, k, v, R.kernel_scale(D, scale), D, causal=True, kernel=True, poly_mask=_poly_mask(D))
        assert not _violates(o.astype(np.float64), lse.astype(np.float64), ref, bound, lb), (gen, scale)
        ne = ~ref["empty"]
        worst = max(worst, (np.abs(o[ne].astype(np.float64) - ref["o"][ne]) / bound[ne]).max())
    assert worst > 0.02, "the bound is far looser than the arithmetic it covers"


def test_empty_rows_are_exact_under_the_kernel_arithmetic():
    """Nq > Nk: the first Nq - Nk rows see no key; the polynomial keys leave l = 2^-126, not 0, and the guard on m
    still gives O = 0 and lse = -inf."""
    D, Nq, Nk = 128, 300, 129
    q, k, v, _ = M.make_inputs("randn", 1, 1, Nq, Nk, D, 64, None, seed=5)
    o, lse = M.online(q[0, 0], k[0, 0], v[0, 0], R.kernel_scale(D), D, causal=True, kernel=True,
                      poly_mask=_poly_mask(D))
    assert np.all(o[:Nq - Nk] == 0) and np.all(lse[:Nq - Nk] == -np.inf)
    assert np.all(np.isfinite(lse[Nq - Nk:]))


@pytest.mark.parametrize("mutation", list(MUTATIONS))
@pytest.mark.parametrize("fam", list(FAMILIES))
def test_mutation_is_rejected(fam, mutation):
    D = FAMILIES[fam]
    caught = []
    for Nq, Nk in SHAPES:
        if mutation == "top_left_alignment" and Nq == Nk:
            continue   # the two alignments agree
        for gen, scale, q, k, v in _cases(D, Nq, Nk):
            ref, bound, lb = _truth(gen, scale, q, k, v)
            o, lse = M.online(q, k, v, R.kernel_scale(D, scale), D, causal=True, **MUTATIONS[mutation])
            if _violates(o, lse, ref, bound, lb):
                caught.append(f"{gen}@{scale} ({Nq},{Nk})")
    assert caught, f"no generator catches {mutation} in family {fam}"
    print(f"{fam}: {mutation} rejected by {', '.join(caught[:6])}{' ...' if len(caught) > 6 else ''}")


def test_probes_pin_the_diagonal():
    """Each probe on its own catches its side of an off-by-one on every shape class."""
    D = 128
    for Nq, Nk in SHAPES:
        for gen, shift in (("diag_gather", -1), ("future_max", 1)):
            q, k, v, _ = M.make_inputs(gen, 1, 1, Nq, Nk, D, 64, None, seed=9)
            q, k, v = q[0, 0], k[0, 0], v[0, 0]
            ref, bound, lb = _truth(gen, None, q, k, v)
            o, lse = M.online(q, k, v, R.kernel_scale(D), D, causal=True, diag_shift=shift)
            assert _violates(o, lse, ref, bound, lb), (gen, Nq, Nk)
