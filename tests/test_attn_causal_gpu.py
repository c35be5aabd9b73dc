"""Causal attention and separate query / key lengths (b200_fmha_fwd_f16_kv) against the masked fp64 reference of
attn_mask_ref.py, element by element within attn_ref's bound, over every kernel family of fmha_dispatch.

Outputs are views inside NaN-pattern guard bands (test_attn_numerics_gpu.py), which must come back bit-identical.
Rows without a visible key (causal, Nq > Nk) must hold O == 0 and lse == -inf exactly.  The largest |err| / bound per
family and shape class is printed at the end of the module (pytest -s).
"""
import collections
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import attn_mask_ref as M
import attn_ref as R
from leetcuda_b200 import _capi, flash_attn
from leetcuda_b200 import merge_attn_states as MA
from test_attn_numerics_gpu import MARGIN, _assert_margins, _guarded

pytestmark = pytest.mark.gpu

HEAD_DIMS = [8, 64, 72, 128, 136, 256, 520]
EQUAL = [(1, 1), (63, 63), (65, 65), (127, 127), (129, 129), (257, 257)]
UNEQUAL = [(1, 777), (16, 2048), (63, 1000), (129, 300), (300, 129), (257, 64)]
_ratios = collections.defaultdict(float)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    if _ratios:
        print("\nlargest |err| / bound (attn_ref.o_bound, lse_bound on the masked reference):")
        for key in sorted(_ratios):
            print(f"  {key[0]:<10} {key[1]:<22} {key[2]:<4} {_ratios[key]:.3f}")


def _shape_class(Nq, Nk, causal):
    cls = "Nq=Nk" if Nq == Nk else ("Nq<Nk" if Nq < Nk else "Nq>Nk")
    return f"{cls} {'causal' if causal else 'full'}"


def _check(got, ref, key, what):
    """O and lse within the bound on the rows that see a key; empty rows exactly O = 0, lse = -inf."""
    o, lse = got
    D = o.shape[-1]
    poly = D <= 128
    _, bound = R.o_bound(ref, poly)
    lb = R.lse_bound(ref, poly)
    empty = ref["empty"]
    if bool(empty.any()):
        assert bool((o[empty] == 0).all()), what + ": O of an empty row is not 0"
        assert bool((lse[empty] == -math.inf).all()), what + ": lse of an empty row is not -inf"
    ne = ~empty
    for name, g, w, b in (("O", o.double(), ref["o"], bound), ("lse", lse.double(), ref["lse"], lb)):
        err = (g[ne] - w[ne]).abs()
        r = torch.nan_to_num(err / b[ne], nan=float("inf"))
        if r.numel() == 0:
            continue
        ratio = r.max().item()
        _ratios[(key[0], key[1], name)] = max(_ratios[(key[0], key[1], name)], ratio)
        if not bool((err <= b[ne]).all()):
            pytest.fail(f"{what} {name}: |err|/bound {ratio:.3g}")


def _run(q, k, v, causal, scale=None, vt=False):
    B, H, Nq, D = q.shape
    obuf, o = _guarded((B, H, Nq, D), torch.float16)
    lbuf, lse = _guarded((B, H, Nq), torch.float32)
    varg = v.transpose(-2, -1).contiguous() if vt else v
    flash_attn.fmha_fwd(q, k, varg, o, v_transposed=vt, scale=scale or 0.0, lse=lse, causal=causal)
    torch.cuda.synchronize()
    _assert_margins(obuf, "O")
    _assert_margins(lbuf, "lse")
    return o, lse


def _case(B, H, Nq, Nk, D, gen, scale, causal, vt=False, seed=0):
    fam, kbn = R.family(D)
    q_np, k_np, v_np, target = M.make_inputs(gen, B, H, Nq, Nk, D, kbn, scale, seed)
    q, k, v = (torch.from_numpy(x).cuda() for x in (q_np, k_np, v_np))
    sc = R.kernel_scale(D, scale)
    what = f"B{B} H{H} Nq{Nq} Nk{Nk} D{D} {gen} scale={scale} causal={causal} vt={vt}"
    o, lse = _run(q, k, v, causal, scale, vt)
    ref = M.reference(q, k, v, sc, causal, exact_scores=M.exact_scores(gen))
    _check((o, lse), ref, (fam, _shape_class(Nq, Nk, causal) + (" vt" if vt else "")), what)
    if gen == "diag_gather" and causal:
        _assert_gather(o, v, target, ~ref["empty"][0, 0].cpu().numpy(), what)


def _assert_gather(o, v, target, rows, what):
    """O[i] = V[target[i]] to within one fp16 ulp on the given rows."""
    truth = v[:, :, torch.from_numpy(target).cuda()].double()
    ulp = torch.exp2(torch.floor(torch.log2(truth.abs().clamp_min(2.0 ** -14))) - 10)
    sel = torch.from_numpy(rows).cuda()
    assert bool(((o.double() - truth).abs() <= ulp)[:, :, sel].all()), what + ": O is not the gathered V"


def _gens(D):
    return [(g, s) for g, s in R.VARIANTS if R.usable(g, D)] + [(p, None) for p in M.PROBES if D >= 32]


@pytest.mark.parametrize("D", HEAD_DIMS)
def test_shape_matrix_causal_equal_lengths(D):
    for Nq, Nk in EQUAL:
        for i, (gen, scale) in enumerate(_gens(D)):
            _case(1, 2, Nq, Nk, D, gen, scale, True, seed=1000 * D + Nq + 7 * i)


@pytest.mark.parametrize("causal", [True, False])
@pytest.mark.parametrize("D", HEAD_DIMS)
def test_shape_matrix_separate_lengths(D, causal):
    for Nq, Nk in UNEQUAL:
        for i, (gen, scale) in enumerate(_gens(D)):
            _case(1, 2, Nq, Nk, D, gen, scale, causal, seed=2000 * D + Nq + 3 * Nk + 7 * i)


@pytest.mark.parametrize("D", [64, 128, 136])
def test_diagonal_probes_across_warpgroups_and_block_edges(D):
    """Diagonals mid-block and on a block edge (diag = Nk - Nq a multiple of kBN or not), with the probe rows in
    both consumer warpgroups of a CTA and in several CTAs."""
    _, kbn = R.family(D)
    for Nq, Nk in [(256, 256), (256, 256 + kbn), (256, 256 + kbn // 2), (192, 192 + 3 * kbn + 1), (320, 100),
                   (200, 200 - kbn)]:
        for gen in M.PROBES:
            for causal in (True, False):
                _case(1, 3, Nq, Nk, D, gen, None, causal, seed=Nq * Nk + D)


@pytest.mark.parametrize("D", [64, 128, 136, 256])
def test_empty_rows(D):
    """Nq > Nk, causal: the first Nq - Nk rows see no key — also whole CTAs of them (nkv = 0) — and must be exactly
    O = 0, lse = -inf; the margins stay intact (checked in _run)."""
    for Nq, Nk in [(300, 1), (1000, 129), (257, 64), (64, 8)]:
        q = torch.randn(2, 2, Nq, D, device="cuda", dtype=torch.half)
        k = torch.randn(2, 2, Nk, D, device="cuda", dtype=torch.half)
        v = torch.randn(2, 2, Nk, D, device="cuda", dtype=torch.half)
        o, lse = _run(q, k, v, True)
        e = Nq - Nk
        assert bool((o[:, :, :e] == 0).all()) and bool((lse[:, :, :e] == -math.inf).all()), (Nq, Nk, D)
        assert bool(torch.isfinite(lse[:, :, e:]).all()) and bool(torch.isfinite(o[:, :, e:]).all()), (Nq, Nk, D)


@pytest.mark.parametrize("D", [72, 128, 136, 264])
def test_transposed_v_separate_lengths(D):
    """V given as [B,H,D,Nk] with Nk != Nq: the vt kernel for D <= 128, the transpose pre-pass for D > 128."""
    for Nq, Nk in [(63, 1000), (300, 136), (129, 64)]:
        for i, (gen, scale) in enumerate(_gens(D)):
            for causal in (True, False):
                _case(1, 2, Nq, Nk, D, gen, scale, causal, vt=True, seed=3000 * D + Nq + 7 * i)


@pytest.mark.parametrize("N,D", [(32768, 128), (16384, 512)])
def test_diag_gather_long_sequence(N, D):
    """Causal diag_gather at long N: the gather is the truth, no N x N reference needed."""
    _, kbn = R.family(D)
    q_np, k_np, v_np, target = M.make_inputs("diag_gather", 1, 1, N, N, D, kbn, None, seed=N + D)
    q, k, v = (torch.from_numpy(x).cuda() for x in (q_np, k_np, v_np))
    o, lse = _run(q, k, v, True)
    _assert_gather(o, v, target, np.ones(N, bool), f"N{N} D{D}")
    # every other visible key is >= 48 nats below: lse = the diagonal score to within lse's own fp32 rounding
    want = (q.double() * k.double()).sum(-1) * R.kernel_scale(D)
    assert bool(((lse.double() - want).abs() <= 2e-6 + 2.0 ** -21 * want.abs() + R.EPS_POLY).all())


def test_grid_limit_heads_causal():
    """B*H = 65535 (the grid.y limit), causal, Nq != Nk: every head's offset against the masked reference."""
    B, H, Nq, Nk, D = 5, 13107, 16, 24, 32
    _case(B, H, Nq, Nk, D, "diag_gather", None, True, seed=65535)


@pytest.mark.parametrize("D", [64, 128, 256])
def test_chunked_prefill_composes_with_merge(D):
    """Queries at positions 768 .. 1023 of a 1024-key sequence: attention over keys [0, 768) (no mask) merged with
    causal attention over [768, 1024), using the kernel's own lse, equals one causal call with Nq = 256, Nk = 1024."""
    H, Nq, Nk, P = 4, 256, 1024, 768
    g = torch.Generator(device="cuda").manual_seed(17 + D)
    q = torch.randn(1, H, Nq, D, device="cuda", dtype=torch.half, generator=g)
    k = torch.randn(1, H, Nk, D, device="cuda", dtype=torch.half, generator=g)
    v = torch.randn(1, H, Nk, D, device="cuda", dtype=torch.half, generator=g)
    sc = R.kernel_scale(D)
    parts = []
    for ks, causal in ((slice(0, P), False), (slice(P, Nk), True)):
        kp, vp = k[:, :, ks].contiguous(), v[:, :, ks].contiguous()
        o, lse = _run(q, kp, vp, causal)
        ref = M.reference(q, kp, vp, sc, causal)
        _check((o, lse), ref, (R.family(D)[0], "chunk part"), f"part {ks}")
        parts.append((o, lse, ref))
    full_o, full_lse = _run(q, k, v, True)
    ref = M.reference(q, k, v, sc, True)
    _check((full_o, full_lse), ref, (R.family(D)[0], "chunk whole"), "whole")
    merged = torch.empty(Nq, H, D, device="cuda", dtype=torch.half)
    merged_lse = torch.empty(H, Nq, device="cuda")
    (oa, la, ra), (ob, lb_, rb) = parts
    MA.merge_attn_states_cuda(merged, oa[0].transpose(0, 1).contiguous(), la[0].contiguous(),
                              ob[0].transpose(0, 1).contiguous(), lb_[0].contiguous(), merged_lse)
    torch.cuda.synchronize()
    # bound: the weighted bounds of the parts, their lse errors through the weights, the merge's fp32 arithmetic and
    # its rounding to fp16
    wa = 1.0 / (1.0 + torch.exp(rb["lse"] - ra["lse"]))[..., None]
    wb = 1.0 - wa
    ba, bb = R.o_bound(ra, D <= 128)[1], R.o_bound(rb, D <= 128)[1]
    dl = (R.lse_bound(ra, D <= 128) + R.lse_bound(rb, D <= 128))[..., None]
    want = ref["o"][0].transpose(0, 1)
    bound = (wa * ba + wb * bb + wa * wb * dl * (ra["o"] - rb["o"]).abs()
             + 2.0 ** -20 * (wa * ra["o"].abs() + wb * rb["o"].abs()) + R.U16 * ref["o"].abs() + 2.0 ** -24)
    bound = bound[0].transpose(0, 1)
    err = (merged.double() - want).abs()
    _ratios[(R.family(D)[0], "chunk merged", "O")] = max(_ratios[(R.family(D)[0], "chunk merged", "O")],
                                                        (err / bound).max().item())
    assert bool((err <= bound).all()), (err / bound).max().item()
    lse_err = (merged_lse.double() - ref["lse"][0]).abs()
    assert bool((lse_err <= R.lse_bound(ref, D <= 128)[0] + R.lse_bound(ra, D <= 128)[0]
                 + R.lse_bound(rb, D <= 128)[0]).all())


@pytest.mark.parametrize("vt", [False, True])
@pytest.mark.parametrize("D", [8, 64, 72, 128, 136, 520])
def test_noncausal_equal_lengths_is_bitwise_the_lse_entry(D, vt):
    """b200_fmha_fwd_f16_kv with causal = 0 and Nq = Nk computes exactly what b200_fmha_fwd_f16_lse computes."""
    for N in (1, 129, 1024):
        if vt and N % 8:
            continue
        q, k, v = (torch.randn(2, 3, N, D, device="cuda", dtype=torch.half) for _ in range(3))
        varg = v.transpose(-2, -1).contiguous() if vt else v
        outs = []
        for entry in ("kv", "lse"):
            o = torch.empty_like(q)
            lse = torch.empty(2, 3, N, device="cuda")
            stream = _capi.raw_stream(q.device.index)
            ptrs = (q.data_ptr(), k.data_ptr(), varg.data_ptr(), o.data_ptr(), lse.data_ptr())
            if entry == "kv":
                rc = _capi.lib().b200_fmha_fwd_f16_kv(*ptrs, 2, 3, N, N, D, int(vt), 0, 0.0, stream)
            else:
                rc = _capi.lib().b200_fmha_fwd_f16_lse(*ptrs, 2, 3, N, D, int(vt), 0.0, stream)
            _capi.check(rc, entry)
            outs.append((o, lse))
        torch.cuda.synchronize()
        assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1]), (D, N, vt)


@pytest.mark.parametrize("D", [64, 128])
def test_sdpa_convention_at_equal_lengths(D):
    """At Nq = Nk the mask is torch SDPA's is_causal (allclose(1e-2, 1e-2), the reference's tolerance)."""
    q, k, v = (torch.randn(2, 4, 1000, D, device="cuda", dtype=torch.half) for _ in range(3))
    o = torch.empty_like(q)
    flash_attn.fmha_fwd(q, k, v, o, causal=True)
    want = F.scaled_dot_product_attention(q, k, v, is_causal=True)
    torch.cuda.synchronize()
    assert torch.allclose(o.float(), want.float(), rtol=1e-2, atol=1e-2)
