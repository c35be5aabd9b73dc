"""The bf16 bound of attn_bf16_ref.py holds for the kernel's bf16 arithmetic and catches the rounding mistakes a bf16
port tends to make.  CPU only (numpy).

The restatement (attn_bf16_ref.online / online_split: fp32 scores and statistics, the polynomial keys, P rounded to
nearest bf16, one rounding of O, or of the combined O on the split path) must stay inside the bound on attn_ref's
generators in every family and on the rounding probes below.  Each mistake, by name, must break it on at least one input:
  * p_truncated       P truncated to bf16 instead of rounded to nearest;
  * inputs_via_fp16   Q, K and V passed through fp16 (values beyond 65504 or below fp16's range);
  * o_truncated       O truncated to bf16;
  * o_rounded_twice   every split's O rounded to bf16 before the combine, then the combined O again.
The rounding probes make the mistakes visible: key 0 scores 0 (P = 1) and the other keys score s with P = exp2(s log2e)
just below a rounding boundary of bf16 (found by a search over bf16 q and k, so the scores are exact in fp32), so that
P's own rounding already uses most of the bound's u sigma term; V is seeded bf16 in [1.02, 1.1), where O's roundings
are worst relative to |O|, one trial per column.
"""
import numpy as np
import pytest

import attn_bf16_ref as BF
import attn_ref as R
import attn_split_ref as SR
from test_attn_bound_sharpness import _poly_mask

FAMILIES = {"D<=64": 64, "64<D<=128": 128, "D>128": 264}
N = 257


def _bf16(x):
    return BF.round_bf16(np.asarray(x, np.float32))


def _variants(D):
    _, kbn = R.family(D)
    for i, (gen, scale) in enumerate(R.VARIANTS):
        if not R.usable(gen, D):
            continue
        q, k, v, _ = R.make_inputs(gen, 1, 1, N, D, kbn, scale, seed=300 + i)
        yield gen, scale, kbn, *(_bf16(x[0, 0].astype(np.float32)) for x in (q, k, v))


def _probe(lo, hi, N=64, D=64, seed=0):
    """(q, k, v) of one head with scale 1: P of keys 1 .. N-1 has the fraction f = P / 2^floor(log2 P) - 1 in
    [lo, hi) (in units of bf16's 2^-7 spacing), key 0 P = 1."""
    c = np.float32(R.LOG2E)
    q0 = _bf16(1.0 + np.arange(128) / 128.0)[:, None]
    k0 = _bf16(-(0.6875 + np.arange(128) / 256.0))[None, :]
    s = (q0 * k0).astype(np.float32)                                  # exact: 8-bit times 8-bit significands
    p = np.exp2((s.astype(np.float64) * np.float64(c)).astype(np.float32)).astype(np.float32)
    f = (p / np.exp2(np.floor(np.log2(p))) - 1) * 128
    i, j = np.argwhere((f >= lo) & (f < hi))[0]
    q = np.zeros((1, D), np.float32)
    k = np.zeros((N, D), np.float32)
    q[0, 0], k[1:, 0] = q0[i, 0], k0[0, j]
    v = _bf16(1.02 + 0.08 * np.random.default_rng(seed).random((N, D)))   # O near 1: roundings of 2^-8 relative
    return q, k, v


PROBES = {"p_rn_down": (0.9 / 2, 0.5), "p_trunc_worst": (0.92, 1.0)}   # f in units of 2^-7


def _truth(q, k, v, scale, exact=False):
    ref = R.reference(q, k, v, scale, exact_scores=exact)
    return ref, BF.o_bound(ref, False)[1] if q.shape[-1] > 128 else None


def _violates(o, want, bound):
    return bool(np.any(np.isnan(o)) or np.any(np.abs(o.astype(np.float64) - want) > bound))


@pytest.mark.parametrize("fam", list(FAMILIES))
def test_kernel_arithmetic_stays_inside_the_bound(fam):
    D = FAMILIES[fam]
    poly = D <= 128
    worst = 0.0
    for gen, scale, kbn, q, k, v in _variants(D):
        sc = R.kernel_scale(D, scale)
        ref = R.reference(q, k, v, sc, exact_scores=gen == "one_hot")
        bound = BF.o_bound(ref, poly)[1]
        o, lse = BF.online(q, k, v, sc, kbn, poly_mask=_poly_mask(D))
        assert not _violates(o, ref["o"], bound), (gen, scale, (np.abs(o - ref["o"]) / bound).max())
        assert np.all(np.abs(lse - ref["lse"]) <= BF.lse_bound(ref, poly)), (gen, scale)
        worst = max(worst, (np.abs(o - ref["o"]) / bound).max())
    assert worst > 0.02, "the bound is far looser than the arithmetic it covers"


def _probe_case(name, seed=0):
    q, k, v = _probe(*PROBES[name], seed=seed)
    ref = R.reference(q, k, v, 1.0)
    return q, k, v, ref, BF.o_bound(ref, False)[1]


@pytest.mark.parametrize("seed", range(4))
@pytest.mark.parametrize("probe", list(PROBES))
def test_kernel_arithmetic_stays_inside_the_bound_on_the_probes(probe, seed):
    q, k, v, ref, bound = _probe_case(probe, seed)
    o, _ = BF.online(q, k, v, 1.0, 64)
    assert not _violates(o, ref["o"], bound), (np.abs(o - ref["o"]) / bound).max()
    parts = SR.part_references(q[None, None], k[None, None], v[None, None], 1.0, False, 2)
    want, _, _, ob, _ = BF.combine_bound(parts, False)
    o2, _ = BF.online_split(q, k, v, 1.0, 32, 2)
    assert not _violates(o2, want[0, 0], ob[0, 0]), (np.abs(o2 - want[0, 0]) / ob[0, 0]).max()


def test_split_arithmetic_stays_inside_the_bound():
    for gen, scale, kbn, q, k, v in _variants(128):
        sc = R.kernel_scale(128, scale)
        parts = SR.part_references(q[None, None], k[None, None], v[None, None], sc, False, 3,
                                   exact_scores=gen == "one_hot")
        want, _, _, ob, _ = BF.combine_bound(parts, True)
        o, _ = BF.online_split(q, k, v, sc, kbn, 3, poly_mask=_poly_mask(128))
        assert not _violates(o, want[0, 0], ob[0, 0]), (gen, scale)


def test_p_truncated_is_rejected():
    q, k, v, ref, bound = _probe_case("p_trunc_worst")
    o, _ = BF.online(q, k, v, 1.0, 64, p_round="rz")
    assert _violates(o, ref["o"], bound)


def test_o_truncated_is_rejected():
    q, k, v, ref, bound = _probe_case("p_rn_down")
    o, _ = BF.online(q, k, v, 1.0, 64, o_round="rz")
    assert _violates(o, ref["o"], bound)


def test_o_rounded_twice_is_rejected():
    """The extra rounding has to meet P's and the final one in the same direction: seeded trials until one does."""
    caught = []
    for seed in range(32):
        q, k, v, _, _ = _probe_case("p_rn_down", seed)
        parts = SR.part_references(q[None, None], k[None, None], v[None, None], 1.0, False, 2)
        want, _, _, ob, _ = BF.combine_bound(parts, False)
        o, _ = BF.online_split(q, k, v, 1.0, 32, 2, part_round="rn")
        if _violates(o, want[0, 0], ob[0, 0]):
            caught.append(seed)
        o, _ = BF.online_split(q, k, v, 1.0, 32, 2)
        assert not _violates(o, want[0, 0], ob[0, 0]), seed
    assert caught
    print(f"o_rounded_twice rejected by seeds {caught}")


def test_inputs_via_fp16_is_rejected():
    """V entries of 1e6 and 1e-30: fp16 makes them inf and 0, bf16 keeps them."""
    caught = []
    for gen, scale, kbn, q, k, v in _variants(128):
        sc = R.kernel_scale(128, scale)
        v = v.copy()
        v[:, 0::2] = _bf16(v[:, 0::2] * 1e6)
        v[:, 1::2] = _bf16(v[:, 1::2] * 1e-30)
        ref = R.reference(q, k, v, sc, exact_scores=gen == "one_hot")
        bound = BF.o_bound(ref, True)[1]
        o, _ = BF.online(q, k, v, sc, kbn, poly_mask=_poly_mask(128))
        assert not _violates(o, ref["o"], bound), gen
        with np.errstate(invalid="ignore", over="ignore"):
            f16 = [x.astype(np.float16).astype(np.float32) for x in (q, k, v)]
            om, _ = BF.online(*f16, sc, kbn, poly_mask=_poly_mask(128))
        if _violates(om, ref["o"], bound):
            caught.append(gen)
    assert caught == [g for g, s, *_ in _variants(128)], caught
