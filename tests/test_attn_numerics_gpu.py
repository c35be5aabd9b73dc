"""Attention against the fp64 reference of attn_ref.py, element by element within its derived bound, over every kernel
family of fmha_dispatch (csrc/attn_capi.cu), both ragged tails, adversarial score distributions and guard bands.

Every call writes O (and lse) into views of larger buffers whose margins hold a fixed NaN bit pattern; the margins must
come back bit-identical, and O / lse must hold no sentinel left over.  With B*H heads laid out back to back, the margin
after the last head is where a store to a row >= N or a column >= D of that head would land.
The largest |err| / bound per kernel family and generator is printed at the end of the module (pytest -s).
"""
import collections

import numpy as np
import pytest
import torch

import attn_ref as R
from leetcuda_b200 import flash_attn, fused_ops

pytestmark = pytest.mark.gpu

HEAD_DIMS = [8, 24, 64, 72, 120, 128, 136, 256, 264, 384, 520, 1024]
SEQ_LENS = [1, 63, 65, 127, 129, 257]
MARGIN = 256                       # elements before and after every output (512 B for fp16: alignment kept)
SENT16, SENT32 = 0x7E5B, 0x7FA5A5A5
RMS_G = 0.75
_ratios = collections.defaultdict(float)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    if _ratios:
        print("\nlargest |err| / bound (attn_ref.o_bound, lse_bound):")
        for key in sorted(_ratios):
            print(f"  {key[0]:<13} {key[1]:<5} {key[2]:<18} {_ratios[key]:.3f}")


def _guarded(shape, dtype):
    n = int(np.prod(shape))
    buf = torch.empty(n + 2 * MARGIN, dtype=dtype, device="cuda")
    if dtype == torch.float16:
        buf.view(torch.int16).fill_(SENT16)
    else:
        buf.view(torch.int32).fill_(SENT32)
    return buf, buf[MARGIN:MARGIN + n].view(shape)


def _assert_margins(buf, what):
    bits = buf.view(torch.int16 if buf.dtype == torch.float16 else torch.int32)
    sent = SENT16 if buf.dtype == torch.float16 else SENT32
    assert bool((bits[:MARGIN] == sent).all()), f"{what}: store before the output"
    assert bool((bits[-MARGIN:] == sent).all()), f"{what}: store past the output"


def _check(got, want, bound, key, what):
    err = (got.double() - want).abs()
    ok = err <= bound                      # NaN (a sentinel never overwritten) fails
    r = torch.nan_to_num(err / bound, nan=float("inf"))
    ratio = r.max().item()
    _ratios[key] = max(_ratios[key], ratio)
    if not bool(ok.all()):
        at = np.unravel_index(int(r.argmax()), tuple(r.shape))
        pytest.fail(f"{what}: |err|/bound {ratio:.3g} at {at}: got {got[at].item()}, want {want[at].item()}")


def _run_case(B, H, N, D, gen, scale, vt=False, rms=False, seed=0):
    fam, kbn = R.family(D, rms)
    q_np, k_np, v_np, perm = R.make_inputs(gen, B, H, N, D, kbn, scale, seed)
    q, k, v = (torch.from_numpy(x).cuda() for x in (q_np, k_np, v_np))
    sc = R.kernel_scale(D, scale)
    ref = R.reference(q, k, v, sc, exact_scores=gen == "one_hot")
    pre, bound = R.o_bound(ref, poly=D <= 128)
    want = ref["o"]
    if rms:
        want, bound = R.rms_reference(ref, RMS_G, pre)
    obuf, o = _guarded((B, H, N, D), torch.float16)
    lbuf, lse = _guarded((B, H, N), torch.float32)
    varg = v.transpose(-2, -1).contiguous() if vt else v
    if rms:
        fused_ops.attn_rmsnorm(q, k, varg, o, RMS_G, v_transposed=vt, scale=scale or 0.0, lse=lse)
    else:
        flash_attn.fmha_fwd(q, k, varg, o, v_transposed=vt, scale=scale or 0.0, lse=lse)
    torch.cuda.synchronize()
    what = f"B{B} H{H} N{N} D{D} {gen} scale={scale} vt={vt} rms={rms}"
    _assert_margins(obuf, what + " O")
    _assert_margins(lbuf, what + " lse")
    label = ("rms " if rms and fam != "rms-cluster" else "") + fam
    tag = "sharp" if scale == 1.0 else ("flat" if scale == 1e-3 else "")
    _check(o, want, bound, (label, "O", f"{gen} {tag}".strip()), what + " O")
    _check(lse, ref["lse"], R.lse_bound(ref, poly=D <= 128), (label, "lse", f"{gen} {tag}".strip()), what + " lse")
    if perm is not None and not rms:
        _assert_gather(o, v, perm, what)


def _assert_gather(o, v, perm, what):
    """O[i] = V[perm[i]] to within one fp16 ulp (the polynomial's exp2(0) = 0.99993 against P rounded to 1.0)."""
    idx = torch.from_numpy(perm).cuda()[..., None].expand(*perm.shape, v.shape[-1])
    truth = torch.gather(v, 2, idx).double()
    ulp = torch.exp2(torch.floor(torch.log2(truth.abs().clamp_min(2.0 ** -14))) - 10)
    assert bool(((o.double() - truth).abs() <= ulp).all()), what + ": O is not the gathered V"


def _variants(D):
    return [(i, g, s) for i, (g, s) in enumerate(R.VARIANTS) if R.usable(g, D)]


def _rms_supported(D):
    return D <= 256 or D in (384, 512)


@pytest.mark.parametrize("N", SEQ_LENS)
@pytest.mark.parametrize("D", HEAD_DIMS)
def test_shape_matrix(D, N):
    """Every family x both tails x every generator, with lse, and the fused RMS norm where the kernel has it."""
    for i, gen, scale in _variants(D):
        _run_case(1, 2, N, D, gen, scale, seed=1000 * D + 10 * N + i)
        if _rms_supported(D):
            _run_case(1, 2, N, D, gen, scale, rms=True, seed=1000 * D + 10 * N + i)


@pytest.mark.parametrize("N", [8, 64, 72, 136, 264])
@pytest.mark.parametrize("D", [24, 72, 128, 136, 264])
def test_transposed_v(D, N):
    """V given as [B,H,D,N]: the vt kernel for D <= 128, the transpose pre-pass for D > 128."""
    for i, gen, scale in _variants(D):
        _run_case(1, 2, N, D, gen, scale, vt=True, seed=7 + 1000 * D + 10 * N + i)


@pytest.mark.parametrize("N,D", [(32768, 128), (16384, 512)])
def test_permutation_recovery_long_sequence(N, D):
    """one_hot at long N, where the gather is the truth and no N x N reference is needed."""
    _, kbn = R.family(D)
    q_np, k_np, v_np, perm = R.make_inputs("one_hot", 1, 1, N, D, kbn, None, seed=N + D)
    q, k, v = (torch.from_numpy(x).cuda() for x in (q_np, k_np, v_np))
    obuf, o = _guarded(q.shape, torch.float16)
    lbuf, lse = _guarded(q.shape[:3], torch.float32)
    flash_attn.fmha_fwd(q, k, v, o, lse=lse)
    torch.cuda.synchronize()
    _assert_margins(obuf, "O")
    _assert_margins(lbuf, "lse")
    _assert_gather(o, v, perm, f"N{N} D{D}")
    # every other key is >= 48 nats below: lse = the winning score to within the fp32 rounding of lse itself
    sc = R.kernel_scale(D)
    win = (q.double() * torch.gather(k, 2, torch.from_numpy(perm).cuda()[..., None].expand(*perm.shape, D)).double())
    want = win.sum(-1) * sc
    assert bool(((lse.double() - want).abs() <= 2e-6 + 2.0 ** -21 * want.abs()).all())


def test_grid_limit_heads():
    """B*H = 65535 (the grid.y limit) at small N: every head's offset, checked against the gather."""
    B, H, N, D = 5, 13107, 16, 32
    q_np, k_np, v_np, perm = R.make_inputs("one_hot", B, H, N, D, 128, None, seed=65535)
    q, k, v = (torch.from_numpy(x).cuda() for x in (q_np, k_np, v_np))
    obuf, o = _guarded(q.shape, torch.float16)
    lbuf, lse = _guarded(q.shape[:3], torch.float32)
    flash_attn.fmha_fwd(q, k, v, o, lse=lse)
    torch.cuda.synchronize()
    _assert_margins(obuf, "O")
    _assert_margins(lbuf, "lse")
    _assert_gather(o, v, perm, "B*H = 65535")
    ref = R.reference(q, k, v, R.kernel_scale(D), exact_scores=True)
    assert bool(((lse.double() - ref["lse"]).abs() <= R.lse_bound(ref, poly=True)).all())
