"""The restated append (kvcache_ref.check_append) accepts the kernel's arithmetic and rejects each wrong design injected
into it: the other rotary pairing, a position off by one, cos and sin swapped, the e4m3 scale multiplied by its
reciprocal instead of divided, no saturation, and a token written one row early.  CPU only."""
import pytest
import torch

import kvcache_ref as K

B, HKV, D, CAP = 3, 2, 64, 64
LENS = [0, 30, 62]


def _setup(T, paged, n_new, e4m3, scale):
    g = torch.Generator().manual_seed(7)
    new = (torch.randn(B, HKV, n_new, D, generator=g) * 3).to(K.TORCH[T])
    if e4m3 and scale < 1:
        new[0, 0, 0, :8] = 200.0   # 200 / scale > 448: the codes saturate
    cos, sin = K.tables(CAP + n_new, D)
    if paged:
        ps, mp = 16, CAP // 16
        num_pages = B * mp + 2
        table = torch.randperm(num_pages, generator=g)[:B * mp].view(B, mp).int()
        rows = num_pages * ps * HKV
        kw = dict(table=table, page_size=ps, num_pages=num_pages)
    else:
        rows, kw = B * HKV * CAP, {}
    dt = torch.float8_e4m3fn if e4m3 else K.TORCH[T]
    before = torch.randint(0, 100, (rows, D), generator=g).to(torch.uint8 if e4m3 else torch.int16).view(dt) \
        if e4m3 else (torch.randn(rows, D, generator=g)).to(dt)
    return new, cos, sin, before, kw


def _run(T, paged, n_new, interleaved, e4m3, scale, mistake):
    new, cos, sin, before, kw = _setup(T, paged, n_new, e4m3, scale)
    after = K.kernel_append(before.clone(), new, LENS, CAP, cos, sin, D, interleaved, T, scale, rotate=True,
                            mistake=mistake, **kw)
    return K.check_append(after, before, new, LENS, CAP, cos, sin, D, interleaved, T, scale, **kw)


@pytest.mark.parametrize("T", K.TYPES)
@pytest.mark.parametrize("paged", [False, True], ids=["dense", "paged"])
@pytest.mark.parametrize("interleaved", [False, True], ids=["neox", "gptj"])
@pytest.mark.parametrize("e4m3", [False, True], ids=["T", "e4m3"])
def test_kernel_arithmetic_passes(T, paged, interleaved, e4m3):
    assert _run(T, paged, 4, interleaved, e4m3, 0.37 if e4m3 else 1.0, None) is None


@pytest.mark.parametrize("T", K.TYPES)
@pytest.mark.parametrize("mistake", ["pairing", "position", "swap", "early"])
@pytest.mark.parametrize("interleaved", [False, True], ids=["neox", "gptj"])
@pytest.mark.parametrize("paged", [False, True], ids=["dense", "paged"])
def test_rotary_and_placement_mistakes_rejected(T, mistake, interleaved, paged):
    assert _run(T, paged, 4, interleaved, False, 1.0, mistake) is not None


def _divide_sensitive(T, scale):
    """Non-negative T values x whose code of x / scale differs from the code of x * fp32(1 / scale)."""
    bits = torch.arange(0, 0x7C00 if T == "half" else 0x7F80, dtype=torch.int32).to(torch.int16)
    x = bits.view(K.TORCH[T])
    differ = K.quantise(x, scale).view(torch.uint8) != K.kernel_quantise(x, scale, "multiply").view(torch.uint8)
    return x[differ]


@pytest.mark.parametrize("T", K.TYPES)
@pytest.mark.parametrize("mistake", ["multiply", "no_saturation", "early"])
def test_e4m3_mistakes_rejected(T, mistake):
    """Without rotary the e4m3 codes must equal quantise() bit for bit: the new rows hold values whose codes change when
    the scale's reciprocal is multiplied (found by searching every T value at scale 7), and 200 / 0.25 = 800, which must
    saturate to 448, not become NaN."""
    for scale in (7.0, 0.25):
        new, cos, sin, before, kw = _setup(T, True, 4, True, scale)
        sens = _divide_sensitive(T, scale)[:D]
        assert scale != 7.0 or sens.numel() > 0
        new[1, 1, 0, :sens.numel()] = sens
        after = K.kernel_append(before.clone(), new, LENS, CAP, cos, sin, 0, False, T, scale, rotate=False,
                                mistake=mistake, **kw)
        if K.check_append(after, before, new, LENS, CAP, cos, sin, 0, False, T, scale, rotate=False, **kw) is not None:
            return
    pytest.fail(f"{mistake} was not caught")


def test_bound_is_tight_for_one_ulp():
    """A rotated value one T spacing away from the kernel's passes only if the bound allows it: moving every rotated
    element by two spacings fails."""
    T = "half"
    new, cos, sin, before, kw = _setup(T, False, 4, False, 1.0)
    after = K.kernel_append(before.clone(), new, LENS, CAP, cos, sin, D, False, T, rotate=True, **kw)
    src, dst = K.cache_rows(B, HKV, 4, LENS, CAP)
    moved = after.clone()
    moved[dst] = (after[dst].double() + 2 * K.ulp(after[dst].double(), T) + 1e-3).to(torch.float16)
    assert K.check_append(moved, before, new, LENS, CAP, cos, sin, D, False, T, **kw) is not None


def test_positions_and_capacity():
    assert K.slot(0, 0, -5, 16) == 0 and K.slot(0, 3, 14, 16) is None and K.slot(0, 1, 14, 16) == 15
    assert K.slot(0, 0, 99, 16) is None                       # clamped to capacity: every token dropped
    table = [[3, -1, 9]]
    assert K.slot(0, 0, 16, 48, table, 16, 9) is None          # entry -1
    assert K.slot(0, 0, 32, 48, table, 16, 9) is None          # entry 9 = num_pages
    assert K.slot(0, 5, 0, 48, table, 16, 9) == (3, 5)
    assert K.seqlens_out([-5, 10, 15, 40], 2, 16) == [2, 12, 16, 16]
