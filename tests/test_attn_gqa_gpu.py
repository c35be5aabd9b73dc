"""Grouped-query attention and split-KV (b200_fmha_fwd_f16_gqa) on the GPU, over every kernel family of fmha_dispatch.

* Without a split, GQA is bit for bit the existing kernel run on K and V with every head repeated (a packed row does the
  same arithmetic on the same key blocks; a fully masked extra block adds 0 to P V and 2^-126 to l >= 1).
* With splits, every element is checked against the fp64 reference on the expanded K/V within attn_split_ref's bound
  of a combined row.  Empty rows must be exactly O = 0, lse = -inf; outputs sit inside NaN guard bands.
"""
import collections
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import attn_mask_ref as M
import attn_ref as R
import attn_split_ref as SR
from leetcuda_b200 import _capi, flash_attn
from test_attn_numerics_gpu import _assert_margins, _guarded

pytestmark = pytest.mark.gpu

HEAD_DIMS = [8, 64, 72, 128, 136, 256, 520]
_ratios = collections.defaultdict(float)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    if _ratios:
        print("\nlargest |err| / bound (attn_split_ref.combine_bound):")
        for key in sorted(_ratios):
            print(f"  {key[0]:<10} {key[1]:<10} {key[2]:<4} {_ratios[key]:.3f}")


def _run(q, k, v, causal, splits, scale=None, vt=False):
    B, H, Nq, D = q.shape
    obuf, o = _guarded((B, H, Nq, D), torch.float16)
    lbuf, lse = _guarded((B, H, Nq), torch.float32)
    varg = v.transpose(-2, -1).contiguous() if vt else v
    flash_attn.fmha_fwd(q, k, varg, o, v_transposed=vt, scale=scale or 0.0, lse=lse, causal=causal,
                        num_splits=splits)
    torch.cuda.synchronize()
    _assert_margins(obuf, "O")
    _assert_margins(lbuf, "lse")
    return o, lse


def _inputs(gen, B, H, Hkv, Nq, Nk, D, scale, seed):
    """attn_mask_ref's generators with Hkv K/V heads.  Queries of one_hot and of the probes are codes of their K/V
    head's keys, so every query head of a group repeats them; the others draw H heads of their own."""
    _, kbn = R.family(D)
    q, k, v, _ = M.make_inputs(gen, B, Hkv, Nq, Nk, D, kbn, scale, seed)
    if gen == "one_hot" or gen in M.PROBES:
        q = np.repeat(q, H // Hkv, axis=1)
    else:
        q = M.make_inputs(gen, B, H, Nq, Nk, D, kbn, scale, seed + 1)[0]
    return (torch.from_numpy(np.ascontiguousarray(x)).cuda() for x in (q, k, v))


# ------------------------------------------------------------------ bitwise without a split
def _expanded(q, k, v, causal, vt):
    G = q.shape[1] // k.shape[1]
    return _run(q, k.repeat_interleave(G, 1).contiguous(), v.repeat_interleave(G, 1).contiguous(), causal, 1, vt=vt)


@pytest.mark.parametrize("D", HEAD_DIMS)
def test_gqa_unsplit_is_bitwise_the_expanded_kernel(D):
    H = 16
    for G in (1, 2, 4, 8, H):
        for Nq, Nk in [(1, 777), (3, 777), (17, 300), (63, 1000), (65, 64), (129, 129), (300, 777), (300, 129)]:
            for causal in (False, True):
                g = torch.Generator(device="cuda").manual_seed(D * 1000 + G * 10 + Nq)
                q = torch.randn(2, H, Nq, D, device="cuda", dtype=torch.half, generator=g)
                k, v = (torch.randn(2, H // G, Nk, D, device="cuda", dtype=torch.half, generator=g) for _ in range(2))
                got = _run(q, k, v, causal, 1)
                want = _expanded(q, k, v, causal, False)
                what = f"D{D} G{G} Nq{Nq} Nk{Nk} causal={causal}"
                assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1]), what


@pytest.mark.parametrize("D", [72, 128, 136, 264])
def test_gqa_unsplit_transposed_v_is_bitwise(D):
    """v_transposed: the vt kernel for D <= 128, the transpose pre-pass over the Hkv heads for D > 128."""
    H, G = 8, 4
    for Nq, Nk in [(1, 776), (17, 136), (129, 64)]:
        for causal in (False, True):
            g = torch.Generator(device="cuda").manual_seed(D + Nq)
            q = torch.randn(1, H, Nq, D, device="cuda", dtype=torch.half, generator=g)
            k, v = (torch.randn(1, H // G, Nk, D, device="cuda", dtype=torch.half, generator=g) for _ in range(2))
            got = _run(q, k, v, causal, 1, vt=True)
            want = _expanded(q, k, v, causal, True)
            assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1]), (D, Nq, Nk, causal)


@pytest.mark.parametrize("D", [64, 128, 256])
def test_mha_through_the_gqa_entry_is_bitwise_the_kv_entry(D):
    B, H, Nq, Nk = 2, 3, 65, 300
    q = torch.randn(B, H, Nq, D, device="cuda", dtype=torch.half)
    k, v = (torch.randn(B, H, Nk, D, device="cuda", dtype=torch.half) for _ in range(2))
    stream = _capi.raw_stream(q.device.index)
    for causal in (0, 1):
        outs = []
        for entry in ("gqa", "kv"):
            o, lse = torch.empty_like(q), torch.empty(B, H, Nq, device="cuda")
            ptrs = (q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), lse.data_ptr())
            if entry == "gqa":
                rc = _capi.lib().b200_fmha_fwd_f16_gqa(*ptrs, B, H, H, Nq, Nk, D, 0, causal, 1, 0.0, stream)
            else:
                rc = _capi.lib().b200_fmha_fwd_f16_kv(*ptrs, B, H, Nq, Nk, D, 0, causal, 0.0, stream)
            _capi.check(rc, entry)
            outs.append((o, lse))
        torch.cuda.synchronize()
        assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1]), (D, causal)


# ------------------------------------------------------------------ fp64 bound with splits
def _check_split(o, lse, q, k, v, sc, causal, splits, exact, key, what):
    parts = SR.part_references(q, k, v, sc, causal, splits, exact)
    want, wl, empty, ob, lb = SR.combine_bound(parts, poly=q.shape[-1] <= 128)
    assert not bool(torch.isnan(o).any()) and not bool(torch.isnan(lse).any()), what + ": NaN"
    if bool(empty.any()):
        assert bool((o[empty] == 0).all()) and bool((lse[empty] == -math.inf).all()), what + ": empty row"
    ne = ~empty
    for name, g, w, b in (("O", o.double(), want, ob), ("lse", lse.double(), wl, lb)):
        err = (g[ne] - w[ne]).abs()
        if err.numel() == 0:
            continue
        ratio = torch.nan_to_num(err / b[ne], nan=float("inf")).max().item()
        _ratios[(key[0], key[1], name)] = max(_ratios[(key[0], key[1], name)], ratio)
        if not bool((err <= b[ne]).all()):
            pytest.fail(f"{what} {name}: |err|/bound {ratio:.3g}")


def _split_counts(Nk, D):
    _, kbn = R.family(D)
    return [2, 3, 7, 0, min(-(-Nk // kbn) + 5, _capi.FMHA_MAX_SPLITS)]   # the last: more than the key blocks


@pytest.mark.parametrize("D", HEAD_DIMS)
def test_split_within_the_combined_bound(D):
    B, H, Hkv = 1, 8, 2
    gens = [(g, s) for g, s in R.VARIANTS if R.usable(g, D)] + [(p, None) for p in M.PROBES if D >= 32]
    i = 0
    for Nk in (1, 63, 777, 8192):
        for Nq in (1, 5, 130):
            if Nk == 8192 and Nq == 130:
                continue
            for causal in (False, True):
                for splits in _split_counts(Nk, D):
                    gen, scale = gens[i % len(gens)]
                    i += 1
                    if gen == "one_hot" and max(Nq, Nk) < 2:
                        gen, scale = "randn", None   # one code cannot outscore another
                    q, k, v = _inputs(gen, B, H, Hkv, Nq, Nk, D, scale, seed=D * 7919 + i)
                    o, lse = _run(q, k, v, causal, splits, scale)
                    S = splits or _auto(B, H, Hkv, Nq, Nk, D)
                    what = f"D{D} Nq{Nq} Nk{Nk} {gen}@{scale} causal={causal} splits={splits}->{S}"
                    _check_split(o, lse, q, k, v, R.kernel_scale(D, scale), causal, S, M.exact_scores(gen),
                                 (R.family(D)[0], "split"), what)


@pytest.mark.parametrize("D", [64, 128, 136])
def test_split_empty_rows_and_empty_splits(D):
    """Nq > Nk, causal: rows without a key and splits without a block; exactly 0 / -inf, margins intact."""
    B, H, Hkv = 2, 4, 1
    for Nq, Nk, splits in [(300, 1, 4), (257, 64, 7), (130, 129, 64)]:
        q = torch.randn(B, H, Nq, D, device="cuda", dtype=torch.half)
        k, v = (torch.randn(B, Hkv, Nk, D, device="cuda", dtype=torch.half) for _ in range(2))
        o, lse = _run(q, k, v, True, splits)
        e = Nq - Nk
        assert bool((o[:, :, :e] == 0).all()) and bool((lse[:, :, :e] == -math.inf).all()), (Nq, Nk, D)
        assert bool(torch.isfinite(lse[:, :, e:]).all()) and bool(torch.isfinite(o[:, :, e:]).all()), (Nq, Nk, D)
        _check_split(o, lse, q, k, v, R.kernel_scale(D), True, splits, False, (R.family(D)[0], "empty"),
                     f"D{D} Nq{Nq} Nk{Nk} splits={splits}")


def _auto(B, H, Hkv, Nq, Nk, D):
    """The split count the library chooses for num_splits = 0 (the bound needs the actual key ranges)."""
    s = _capi.lib().b200_fmha_fwd_f16_gqa_splits(B, H, Hkv, Nq, Nk, D)
    assert 1 <= s <= _capi.FMHA_MAX_SPLITS, s
    return s


# ------------------------------------------------------------------ long decode gather
@pytest.mark.parametrize("Nk", [65536, 65500])
def test_long_decode_gather(Nk):
    """q = a scaled one-hot code of one key (>= 48 nats above every other key): O is that V row to one fp16 ulp.
    Targets in the middle of a split, on both sides of a split boundary and in the last (ragged) block."""
    D, H, Hkv = 128, 8, 2
    G = H // Hkv
    _, kbn = R.family(D)
    _, k_np, v_np, _ = R.make_inputs("one_hot", 1, Hkv, Nk, D, kbn, None, seed=Nk)
    k, v = torch.from_numpy(k_np).cuda(), torch.from_numpy(v_np).cuda()
    c = np.float16(24.0 / R.kernel_scale(D))
    num_kv = -(-Nk // kbn)
    for Nq in (1, 2, 3, 4):
        for splits in (0, 7):
            S = splits or _auto(1, H, Hkv, Nq, Nk, D)
            b1 = num_kv // S   # first block of split 1
            cand = [b1 * kbn // 2, b1 * kbn - 1, b1 * kbn, (num_kv * 2 // S) * kbn + 17, (num_kv - 1) * kbn + 1,
                    Nk - Nq]
            # every target is visible to every position under the causal mask (key <= Nk - Nq)
            target = np.array([[min(cand[(h + 3 * i) % len(cand)], Nk - Nq) for i in range(Nq)] for h in range(H)])
            q_np = np.stack([k_np[0, h // G, target[h]] for h in range(H)])[None].astype(np.float32) * np.float32(c)
            q = torch.from_numpy(q_np.astype(np.float16)).cuda()
            for causal in (False, True):
                o, lse = _run(q, k, v, causal, splits)
                truth = torch.stack([v[0, h // G, torch.from_numpy(target[h]).cuda()] for h in range(H)])[None]
                truth = truth.double()
                ulp = torch.exp2(torch.floor(torch.log2(truth.abs().clamp_min(2.0 ** -14))) - 10)
                assert bool(((o.double() - truth).abs() <= ulp).all()), (Nk, Nq, splits, causal)


# ------------------------------------------------------------------ launches and convention
def test_launch_count():
    q = torch.randn(1, 8, 1, 128, device="cuda", dtype=torch.half)
    k, v = (torch.randn(1, 2, 4096, 128, device="cuda", dtype=torch.half) for _ in range(2))
    o = torch.empty_like(q)
    for splits, launches in ((1, 1), (4, 2), (64, 2)):
        torch.cuda.synchronize()
        n0 = _capi.launch_count()
        flash_attn.fmha_fwd(q, k, v, o, num_splits=splits)
        assert _capi.launch_count() - n0 == launches, splits
    n0 = _capi.launch_count()
    flash_attn.fmha_fwd(q, k, v, o, num_splits=0)
    assert _capi.launch_count() - n0 in (1, 2)
    torch.cuda.synchronize()


@pytest.mark.parametrize("splits", [1, 0, 3])
@pytest.mark.parametrize("D", [64, 128])
def test_sdpa_enable_gqa_convention(D, splits):
    """At Nq = Nk the head mapping and mask are torch SDPA's enable_gqa (allclose(1e-2, 1e-2), the reference's
    tolerance)."""
    q = torch.randn(2, 8, 1000, D, device="cuda", dtype=torch.half)
    k, v = (torch.randn(2, 2, 1000, D, device="cuda", dtype=torch.half) for _ in range(2))
    for causal in (False, True):
        o = torch.empty_like(q)
        flash_attn.fmha_fwd(q, k, v, o, causal=causal, num_splits=splits)
        want = F.scaled_dot_product_attention(q, k, v, is_causal=causal, enable_gqa=True)
        torch.cuda.synchronize()
        assert torch.allclose(o.float(), want.float(), rtol=1e-2, atol=1e-2), (D, splits, causal)
