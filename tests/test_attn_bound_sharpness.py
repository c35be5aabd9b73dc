"""The attention error bound of attn_ref.py is sharp enough to catch the mistakes a kernel rewrite tends to make, and
loose enough for the kernel's own arithmetic.  CPU only (numpy), at small shapes of every kernel family.

For each family, every mutation below applied to the fp64 online softmax must break the bound on at least one of the
inputs the GPU tests use for that family (attn_ref.VARIANTS); a restatement of the kernel's arithmetic (fp32 statistics,
P rounded to fp16, the polynomial keys of B200_ATTN_POLY_MASK, fp16 output) must stay inside it on all of them.
"""
import re
from pathlib import Path

import numpy as np
import pytest

import attn_ref as R

SRC = Path(__file__).resolve().parents[1] / "leetcuda_b200" / "csrc" / "attn_sm90.cuh"
# family -> (D, N): N = 257 gives several key blocks and a ragged last block of one key in every family
SHAPES = {"D<=64": (64, 257), "64<D<=128": (128, 257), "D>128": (264, 257), "rms-cluster": (384, 257)}
RMS_G = 0.75


def _poly_mask(D):
    masks = dict(re.findall(r"#define (B200_ATTN_POLY_MASK(?:_D64)?) (0x[0-9a-fA-F]+)u", SRC.read_text()))
    assert len(masks) == 2
    if D <= 64:
        return int(masks["B200_ATTN_POLY_MASK_D64"], 16)
    return int(masks["B200_ATTN_POLY_MASK"], 16) if D <= 128 else 0


def _swap_keys(k, v):
    v = v.copy()
    v[[3, 12]] = v[[12, 3]]                # keys 3 and 12 of the first 16-key group: P of one meets V of the other
    return k, v


def _slab1_reads_slab0(k, v):
    v = v.copy()
    v[:, 256:] = v[:, :v.shape[1] - 256]   # the second 256-column slab of O computed from the first columns of V
    return k, v


def _leak_zero_key(k, v):
    z = np.zeros((1, k.shape[1]), k.dtype)
    return np.concatenate([k, z]), np.concatenate([v, z])   # the key past N that TMA zero-fills


MUTATIONS = {
    "leaked_zero_key": (_leak_zero_key, None),
    "last_key_dropped": (lambda k, v: (k[:-1], v[:-1]), None),
    "block_rescale_skipped": (lambda k, v: (k, v), 1),
    "p_v_keys_swapped": (_swap_keys, None),
    "slab1_reads_slab0_columns": (_slab1_reads_slab0, None),
}


def _cases(fam):
    D, N = SHAPES[fam]
    _, kbn = R.family(D, rms=fam == "rms-cluster")
    for i, (gen, scale) in enumerate(R.VARIANTS):
        if not R.usable(gen, D):
            continue
        q, k, v, _ = R.make_inputs(gen, 1, 1, N, D, kbn, scale, seed=100 + i)
        yield gen, scale, kbn, q[0, 0], k[0, 0], v[0, 0]


def _truth(fam, gen, scale, q, k, v):
    """(reference output, its bound, lse, lse bound)."""
    D = q.shape[-1]
    sc = R.kernel_scale(D, scale)
    ref = R.reference(q, k, v, sc, exact_scores=gen == "one_hot")
    poly = D <= 128
    pre, bound = R.o_bound(ref, poly)
    out = ref["o"]
    if fam == "rms-cluster":
        out, bound = R.rms_reference(ref, RMS_G, pre)
    return out, bound, ref["lse"], R.lse_bound(ref, poly)


@pytest.mark.parametrize("fam", list(SHAPES))
def test_kernel_arithmetic_stays_inside_the_bound(fam):
    D, _ = SHAPES[fam]
    worst = 0.0
    for gen, scale, kbn, q, k, v in _cases(fam):
        want, bound, lse64, lb = _truth(fam, gen, scale, q, k, v)
        got, lse = R.online(q, k, v, R.kernel_scale(D, scale), kbn, kernel=True, poly_mask=_poly_mask(D),
                            rms_g=RMS_G if fam == "rms-cluster" else 0.0)
        err = np.abs(got.astype(np.float64) - want)
        assert np.all(err <= bound), (gen, scale, (err / bound).max())
        assert np.all(np.abs(lse - lse64) <= lb), (gen, scale)
        worst = max(worst, (err / bound).max())
    assert worst > 0.02, "the bound is far looser than the arithmetic it covers"


@pytest.mark.parametrize("mutation", list(MUTATIONS))
@pytest.mark.parametrize("fam", list(SHAPES))
def test_mutation_is_rejected(fam, mutation):
    D, _ = SHAPES[fam]
    if mutation == "slab1_reads_slab0_columns" and D <= 256:
        pytest.skip("one column slab")
    mutate, skip_block = MUTATIONS[mutation]
    caught = []
    for gen, scale, kbn, q, k, v in _cases(fam):
        want, bound, _, _ = _truth(fam, gen, scale, q, k, v)
        km, vm = mutate(k, v)
        got, _ = R.online(q, km, vm, R.kernel_scale(D, scale), kbn, skip_alpha_block=skip_block,
                          rms_g=RMS_G if fam == "rms-cluster" else 0.0)
        if np.any(np.abs(got - want) > bound):
            caught.append(f"{gen}@{scale}")
    assert caught, f"no generator catches {mutation} in family {fam}"
    print(f"{fam}: {mutation} rejected by {', '.join(caught)}")
