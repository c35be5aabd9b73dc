"""The GEMM kernels against the fp64 reference of gemm_ref.py, element by element within each mode's derived bound (or
bit for bit for the probes), over all ten instantiations of hgemm_wgmma_kernel, both B layouts, ragged M, N and K,
persistent CTAs running several tiles, partial raster groups, the fp16 conversion edges, the TF32 rounding pass and
the peer-store epilogue of the fused all-gather.

Every call writes C into a view of a larger buffer whose margins hold a NaN bit pattern; the margins must come back
bit-identical.  Inputs the mode promises not to touch must come back bit-identical too.
The largest |err| / bound per mode, layout and generator is printed at the end of the module (pytest -s).
"""
import collections
import ctypes

import numpy as np
import pytest
import torch

import gemm_ref as R
from leetcuda_b200 import _capi, hgemm, sgemm
from oracle import oracle as O

pytestmark = pytest.mark.gpu

MARGIN = 256                       # elements before and after every C (alignment kept)
SENT16, SENT32 = 0x7E5B, 0x7FA5A5A5
# (mode, B given as [N,K] storage).  TF32 has one instantiation per tile width; [K,N] B is transposed first.
CALLS = [("f16", False), ("f16", True), ("f16acc", False), ("f16acc", True),
         ("tf32", False), ("tf32", True), ("tf32t", False), ("tf32t", True), ("3xtf32", False)]
# M x N x K (fp16 K; TF32 runs TF32_K[K] instead).  On 132 SMs (see test_shape_table_coverage):
#   2600 x 2000 x 136   128-column tile, 336 tiles, 3 per CTA, tiles_m = 21: a partial, odd group walking n backwards
#   2600 x 2344 x 136   256-column tile, 210 tiles, 2 per CTA, N tail of 40
#   2600 x 2344 x 8     the same tiles with one k-block each
#   8192 x 4096 x 8     256-column tile, one k-block per tile, 8 tiles per CTA: the 4-slot mbarrier ring wraps across
#                       tiles, so the producer waits on a slot the consumers released after a single-k-block tile
#   8576 x 1416 x 8     the same at the 128-column tile: 804 tiles, 7 per CTA through a 6-slot ring
#   3000 x 120 x 4096   256-column tile (N <= 128: equal tile counts, the 0.9 factor keeps 256), long K
#   and small edges.
SHAPES = [(2600, 2000, 136), (2600, 2344, 136), (2600, 2344, 8), (8192, 4096, 8), (8576, 1416, 8),
          (3000, 120, 4096), (1, 8, 8), (7, 24, 8), (65, 136, 72), (127, 264, 200)]
TF32_K = {136: 132, 8: 4, 72: 36}
LAUNCHES = {("f16", False): 1, ("f16", True): 1, ("f16acc", False): 1, ("f16acc", True): 1,
            ("tf32", False): 3, ("tf32", True): 3, ("tf32t", False): 2, ("tf32t", True): 1, ("3xtf32", False): 3}
_ratios = collections.defaultdict(float)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    if _ratios:
        print("\nlargest |err| / bound (gemm_ref.bound):")
        for key in sorted(_ratios):
            print(f"  {key[0]:<7} {key[1]:<3} {key[2]:<10} {_ratios[key]:.3f}")


def _k(mode, K):
    return K if R.is_fp16(mode) else TF32_K.get(K, K)


def _guarded(shape, dtype):
    n = int(np.prod(shape))
    buf = torch.empty(n + 2 * MARGIN, dtype=dtype, device="cuda")
    if dtype == torch.float16:
        buf.view(torch.int16).fill_(SENT16)
    else:
        buf.view(torch.int32).fill_(SENT32)
    return buf, buf[MARGIN:MARGIN + n].view(shape)


def _bits(t):
    return t.view(torch.int16 if t.dtype == torch.float16 else torch.int32)


def _untouched(t):
    return bool((_bits(t) == (SENT16 if t.dtype == torch.float16 else SENT32)).all())


def _assert_margins(buf, what):
    assert _untouched(buf[:MARGIN]), f"{what}: store before C"
    assert _untouched(buf[-MARGIN:]), f"{what}: store past C"


def _check(got, a, b, mode, key, what, info=None):
    """got (device) against the reference of the logical operands a [M,K], b [K,N] (device, as given)."""
    ref = R.reference(a, b, mode)
    bound = R.bound(ref)
    if info is not None:
        want = ref["c"]
        if not torch.equal(got.double(), want):
            pytest.fail(f"{what}: " + R.probe_miss(a.cpu().numpy(), b.cpu().numpy(), got.cpu().double().numpy(),
                                                    want.cpu().numpy(), info))
        return
    err = (got.double() - ref["c"]).abs()
    r = torch.nan_to_num(err / bound, nan=float("inf"))
    ratio = r.max().item()
    _ratios[key] = max(_ratios[key], ratio)
    if not bool((err <= bound).all()):
        at = np.unravel_index(int(r.argmax()), tuple(r.shape))
        pytest.fail(f"{what}: |err|/bound {ratio:.3g} at {at}: got {got[at].item()}, want {ref['c'][at].item()}")


def _call(mode, tn, a, b, c):
    """Run one mode; b is the logical [K,N] operand, passed as a copy ([N,K] storage when tn), so that b itself stays
    the unchanged original.  Returns the B tensor passed."""
    K, N = b.shape
    if R.is_fp16(mode):
        barg = b.t().reshape(K, N).contiguous() if tn else b.clone()
        hgemm.hgemm(a, barg, c, tn=tn, acc="f16" if mode == "f16acc" else "f32")
    elif mode == "3xtf32":
        barg = b.clone()
        sgemm.sgemm_3xtf32(a, barg, c)
    else:
        barg = b.t().contiguous().view(K, N) if tn else b.clone()
        sgemm.sgemm_tf32(a, barg, c, tn=tn, round_inputs=mode == "tf32")
    return barg


def _logical(barg, tn):
    K, N = barg.shape
    return barg.view(N, K).t() if tn else barg


@pytest.mark.parametrize("gen", R.GENERATORS)
@pytest.mark.parametrize("shape", SHAPES, ids=[f"{m}x{n}x{k}" for m, n, k in SHAPES])
def test_shape_matrix(shape, gen):
    """Every mode x layout on one shape and generator: each output within its bound (probes: bit-exact), guard bands
    intact, inputs untouched where the mode promises it (in-place TF32 rounding: exactly tf32(input))."""
    M, N, K0 = shape
    inputs = {}
    for mode, tn in CALLS:
        K = _k(mode, K0)
        dt = np.float16 if R.is_fp16(mode) else np.float32
        if (dt, K) not in inputs:
            a_np, b_np, info = R.make_inputs(gen, M, N, K, dt, seed=M + 7 * N + 31 * K + 1000 * R.GENERATORS.index(gen))
            inputs[(dt, K)] = (torch.from_numpy(a_np).cuda(), torch.from_numpy(b_np).cuda(), info)
        a0, b0, info = inputs[(dt, K)]
        a = a0.clone()
        buf, c = _guarded((M, N), torch.float16 if R.is_fp16(mode) else torch.float32)
        before = _capi.launch_count()
        barg = _call(mode, tn, a, b0, c)
        torch.cuda.synchronize()
        what = f"{M}x{N}x{K} {gen} {mode} {'TN' if tn else 'NN'}"
        assert _capi.launch_count() - before == LAUNCHES[(mode, tn)], what
        _assert_margins(buf, what)
        b_after = _logical(barg, tn)
        a_want, b_want = (R.tf32(a0), R.tf32(b0)) if mode == "tf32" else (a0, b0)
        assert torch.equal(_bits(a), _bits(a_want)) and torch.equal(_bits(b_after.contiguous()), _bits(b_want)), what
        _check(c, a0, b0, mode, (mode, "TN" if tn else "NN", gen), what, info if gen in R.EXACT else None)


def test_shape_table_coverage():
    """On 132 SMs the shape table reaches all ten kernel instantiations, each with more than one tile per CTA, a
    partial raster group, an odd group (n-tiles walked backwards), ragged M, N and K, K below one k-block, and tiles
    of a single k-block each on a CTA that runs more of them than the smem ring has slots, so that the ring wraps
    across tiles."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    if sms != 132:
        pytest.skip(f"the table is laid out for 132 SMs, this device has {sms}")
    multi, seen = set(), set()
    wrapped = set()
    partial_odd = short_k = False
    for M, N, K0 in SHAPES:
        t = R.tile_width(M, N, sms)
        for mode, tn in CALLS:
            K = _k(mode, K0)
            inst = R.instantiation(mode, tn, t["bn"])
            seen.add(inst)
            kblocks = -(-K // R.KBLOCK[mode])
            if t["tiles_per_cta"] > 1:
                multi.add(inst)
            if kblocks == 1 and t["tiles_per_cta"] * kblocks > R.STAGES[t["bn"]]:
                wrapped.add(inst)
            short_k |= K < R.KBLOCK[mode]
        partial_odd |= any(gm < R.GROUP_M and back for _, gm, back in t["groups"])
    def name(inst):
        return "hgemm_wgmma_kernel<%d, %s, %s, %s>" % (inst[0], *(str(x).lower() for x in inst[1:]))
    assert sorted(map(name, R.ALL_INSTANTIATIONS)) == [
        "hgemm_wgmma_kernel<128, false, false, false>", "hgemm_wgmma_kernel<128, false, false, true>",
        "hgemm_wgmma_kernel<128, false, true, false>", "hgemm_wgmma_kernel<128, true, false, false>",
        "hgemm_wgmma_kernel<128, true, false, true>", "hgemm_wgmma_kernel<256, false, false, false>",
        "hgemm_wgmma_kernel<256, false, false, true>", "hgemm_wgmma_kernel<256, false, true, false>",
        "hgemm_wgmma_kernel<256, true, false, false>", "hgemm_wgmma_kernel<256, true, false, true>"]
    assert seen == multi == R.ALL_INSTANTIATIONS, "not run with several tiles per CTA: " + ", ".join(
        sorted(map(name, R.ALL_INSTANTIATIONS - multi)))
    assert wrapped == R.ALL_INSTANTIATIONS, "no single-k-block ring wrap: " + ", ".join(
        sorted(map(name, R.ALL_INSTANTIATIONS - wrapped)))
    assert partial_odd and short_k
    assert any(M % 128 and N % 8 == 0 and N % 128 and K0 % 64 for M, N, K0 in SHAPES)


# ------------------------------------------------------------------ headline sizes, sampled rows
def _sample_rows(M):
    """64 distinct rows spread over all row tiles (two per tile at M = 4096), at varying offsets inside their tile."""
    i = np.arange(64)
    rows = i * (M // 128) // 64 * 128 + (i * 37) % 128
    assert len(np.unique(rows)) == 64
    return torch.from_numpy(rows).cuda()


@pytest.mark.parametrize("mode", ["f16", "f16acc"])
def test_fp16_headline_8192(mode):
    S = 8192
    g = torch.Generator(device="cuda").manual_seed(81)
    a = torch.randn(S, S, device="cuda", dtype=torch.half, generator=g)
    b = torch.randn(S, S, device="cuda", dtype=torch.half, generator=g)
    buf, c = _guarded((S, S), torch.half)
    hgemm.hgemm(a, b, c, acc="f16" if mode == "f16acc" else "f32")
    torch.cuda.synchronize()
    _assert_margins(buf, f"8192^3 {mode}")
    rows = _sample_rows(S)
    _check(c[rows], a[rows], b, mode, (mode, "NN", "randn 8192"), f"8192^3 {mode}")


def test_tf32_headline_8192_bench_op():
    """The bench's SGEMM row: the reference-facing op rounds a, b in place, then the 256-wide tile runs 16 tiles per
    CTA at 32-element k-blocks."""
    S = 8192
    g = torch.Generator(device="cuda").manual_seed(82)
    a0 = torch.randn(S, S, device="cuda", generator=g)
    b0 = torch.randn(S, S, device="cuda", generator=g)
    a, b = a0.clone(), b0.clone()
    buf, c = _guarded((S, S), torch.float32)
    sgemm.sgemm_wmma_m16n16k8_mma4x2_warp2x4_stages(a, b, c, 2, False, 1)
    torch.cuda.synchronize()
    _assert_margins(buf, "tf32 8192^3")
    assert torch.equal(_bits(a), _bits(R.tf32(a0))) and torch.equal(_bits(b), _bits(R.tf32(b0)))
    rows = _sample_rows(S)
    _check(c[rows], a0[rows], b0, "tf32", ("tf32", "NN", "randn 8192"), "tf32 8192^3")


def test_3xtf32_headline_4096():
    S = 4096
    g = torch.Generator(device="cuda").manual_seed(83)
    a = torch.randn(S, S, device="cuda", generator=g)
    b = torch.randn(S, S, device="cuda", generator=g)
    a0, b0 = a.clone(), b.clone()
    buf, c = _guarded((S, S), torch.float32)
    sgemm.sgemm_3xtf32(a, b, c)
    torch.cuda.synchronize()
    _assert_margins(buf, "3xtf32 4096^3")
    assert torch.equal(_bits(a), _bits(a0)) and torch.equal(_bits(b), _bits(b0))
    rows = _sample_rows(S)
    _check(c[rows], a[rows], b, "3xtf32", ("3xtf32", "NN", "randn 4096"), "3xtf32 4096^3")


# ------------------------------------------------------------------ fp16 conversion edges
@pytest.mark.parametrize("tn", [False, True])
@pytest.mark.parametrize("mode", ["f16", "f16acc"])
def test_fp16_overflow_edge(mode, tn):
    """Exact integer sums: 65504 (the largest fp16) and 65519 stay finite at 65504, 65520 and above become +-inf."""
    K, N = 16, 8
    sums = [65504, 65519, 65520, 65536, 98304, 1000]
    a = torch.zeros(2 * len(sums), K)
    b = torch.zeros(K, N)
    b[0, :], b[1, :] = 32, 1                      # C[r, :] = 32 a[r, 0] + a[r, 1]
    for i, v in enumerate(sums):
        for j, sgn in enumerate((1, -1)):
            a[2 * i + j, 0], a[2 * i + j, 1] = sgn * (v // 32), sgn * (v % 32)
    a, b = a.half().cuda(), b.half().cuda()
    buf, c = _guarded((a.shape[0], N), torch.half)
    _call(mode, tn, a, b, c)
    torch.cuda.synchronize()
    _assert_margins(buf, "overflow edge")
    want = torch.tensor([[s * v] for v in sums for s in (1, -1)], dtype=torch.float32).expand(-1, N).cuda()
    want = torch.where(want.abs() >= 65520, want.sign() * float("inf"), torch.clamp(want, -65504, 65504))
    assert torch.equal(c.float(), want), c[:, 0].tolist()


@pytest.mark.parametrize("tn", [False, True])
@pytest.mark.parametrize("mode", ["f16", "f16acc"])
def test_fp16_subnormal_outputs_exact(mode, tn):
    """Integer multiples of 2^-12 in A and B: every partial sum lies on the 2^-24 grid below 2^-14, so C is an fp16
    subnormal (or zero) computed exactly."""
    M, N, K = 256, 264, 16
    g = torch.Generator(device="cuda").manual_seed(84)
    a = (torch.randint(-7, 8, (M, K), device="cuda", generator=g) * 2.0 ** -12).half()
    b = (torch.randint(-7, 8, (K, N), device="cuda", generator=g) * 2.0 ** -12).half()
    buf, c = _guarded((M, N), torch.half)
    _call(mode, tn, a, b, c)
    torch.cuda.synchronize()
    _assert_margins(buf, "subnormal outputs")
    want = a.double() @ b.double()
    assert bool((want.abs() < 2.0 ** -14).all()) and (want != 0).float().mean().item() > 0.9
    assert torch.equal(c.double(), want)


# ------------------------------------------------------------------ TF32 rounding pass, bit for bit
def _round_on_device(x_np, n=None, pad=0):
    """b200_tf32_round_inplace on the first n elements of a device copy of x_np (plus `pad` guard elements)."""
    n = x_np.size if n is None else n
    buf = torch.empty(x_np.size + pad, dtype=torch.float32, device="cuda")
    _bits(buf).fill_(SENT32)
    buf[:x_np.size] = torch.from_numpy(x_np).cuda()
    rc = _capi.lib().b200_tf32_round_inplace(buf.data_ptr(), n, torch.cuda.current_stream().cuda_stream)
    assert rc == 0, _capi.last_error()
    torch.cuda.synchronize()
    return buf.cpu().numpy()


def test_tf32_round_capped_grid():
    """8192^2 floats: more than 16 CTAs per SM would be needed, so the grid is capped and each thread makes many
    grid-stride passes."""
    x = np.random.default_rng(85).standard_normal(8192 * 8192, dtype=np.float32)
    assert x.size / 4 > 16 * torch.cuda.get_device_properties(0).multi_processor_count * 256 * 4
    got = _round_on_device(x)
    assert np.array_equal(got.view(np.uint32), O.tf32_round(x).view(np.uint32))


@pytest.mark.parametrize("n", [1, 2, 3, 4 * 1000 + 1, 4 * 1000 + 2, 4 * 1000 + 3, 4 * 300000 + 3])
def test_tf32_round_tail(n):
    """n % 4 != 0: the scalar tail is rounded and the element after n is not touched."""
    x = np.random.default_rng(n).standard_normal(n + 5, dtype=np.float32)
    got = _round_on_device(x, n=n)
    assert np.array_equal(got[:n].view(np.uint32), O.tf32_round(x[:n]).view(np.uint32))
    assert np.array_equal(got[n:n + 5].view(np.uint32), x[n:].view(np.uint32))


def test_tf32_round_special_values():
    """+-0, subnormals, +-inf, NaN payloads, the largest finite float and rounding ties against oracle.tf32_round
    (cvt.rna.tf32.f32 is the truth).  The bits the device produced are printed for the record."""
    special = np.array([0x00000000, 0x80000000, 0x00000001, 0x80000001, 0x00000FFF, 0x00001000, 0x00001FFF,
                        0x007FFFFF, 0x807FFFFF, 0x00800000, 0x7F7FFFFF, 0xFF7FFFFF, 0x7F7FEFFF, 0x7F800000,
                        0xFF800000, 0x7FC00000, 0xFFC00000, 0x7FC01234, 0x7F800001, 0x7FFFFFFF, 0x3F801000,
                        0xBF801000, 0x3F803000, 0x3F800FFF], np.uint32)
    x = np.tile(special, 4)[:-1].view(np.float32)  # through the float4 body and the scalar tail
    got = _round_on_device(x).view(np.uint32)
    want = O.tf32_round(x).view(np.uint32)
    print("\ncvt.rna.tf32.f32:", " ".join(f"{i:08x}->{o:08x}" for i, o in zip(special, got[:special.size])))
    diff = [(f"{i:08x}", f"{g:08x}", f"{w:08x}") for i, g, w in zip(x.view(np.uint32), got, want) if g != w]
    assert not diff, diff


# ------------------------------------------------------------------ peer-store epilogue on one GPU
ROWS, FN, FK, ROW0, MTOT = 200, 264, 136, 77, 300


def _fused(a, barg, c, peers, n_peers, tn, mc=None, row0=ROW0, peer_array=True):
    arr = (ctypes.c_void_p * max(len(peers), 1))(*[p.data_ptr() for p in peers]) if peer_array else None
    return _capi.lib().b200_hgemm_f16_rows_fused(
        a.data_ptr(), barg.data_ptr(), c.data_ptr(), mc, arr, n_peers, a.shape[0], FN, FK,
        _capi.B_ROW_MAJOR_NK if tn else _capi.B_ROW_MAJOR_KN, row0, torch.cuda.current_stream().cuda_stream)


def _fused_inputs(tn):
    a_np, b_np, _ = R.make_inputs("randn", ROWS, FN, FK, np.float16, seed=86)
    a, b = torch.from_numpy(a_np).cuda(), torch.from_numpy(b_np).cuda()
    return a, b, (b.t().reshape(FK, FN).contiguous() if tn else b)


@pytest.mark.parametrize("direct_env", [False, True])
@pytest.mark.parametrize("n_peers", [1, 3, 7])
@pytest.mark.parametrize("tn", [False, True])
def test_fused_epilogue_peer_stores(tn, n_peers, direct_env, monkeypatch):
    """Local buffers stand in for the peer GPUs' C: every one receives the shard rows bit for bit and nothing else.
    With B200_FUSED_EPILOGUE=direct but no multicast mapping the peers are still used."""
    if direct_env:
        monkeypatch.setenv("B200_FUSED_EPILOGUE", "direct")
    a, b, barg = _fused_inputs(tn)
    bufs = [_guarded((MTOT, FN), torch.half) for _ in range(n_peers + 1)]
    (cbuf, c), peers = bufs[0], [v for _, v in bufs[1:]]
    before = _capi.launch_count()
    assert _fused(a, barg, c, peers, n_peers, tn) == 0, _capi.last_error()
    torch.cuda.synchronize()
    assert _capi.launch_count() - before == 1
    shard = c[ROW0:ROW0 + ROWS]
    _check(shard, a, b, "f16", ("f16", "TN" if tn else "NN", "fused"), "fused epilogue")
    for i, (buf, view) in enumerate(bufs):
        assert torch.equal(_bits(view[ROW0:ROW0 + ROWS]), _bits(shard)), f"peer {i - 1}: shard rows differ from C"
        assert _untouched(buf[:MARGIN + ROW0 * FN]) and _untouched(buf[MARGIN + (ROW0 + ROWS) * FN:]), \
            f"buffer {i}: store outside the shard rows"


@pytest.mark.parametrize("case", ["8_peers", "null_peer_array", "no_target", "negative_row0"])
def test_fused_epilogue_rejects_bad_arguments(case):
    a, b, barg = _fused_inputs(False)
    bufs = [_guarded((MTOT, FN), torch.half) for _ in range(9)]
    c, peers = bufs[0][1], [v for _, v in bufs[1:]]
    kw = {"8_peers": dict(n_peers=8), "null_peer_array": dict(n_peers=3, peer_array=False),
          "no_target": dict(n_peers=0), "negative_row0": dict(n_peers=3, row0=-1)}[case]
    before = _capi.launch_count()
    rc = _fused(a, barg, c, peers, tn=False, **kw)
    torch.cuda.synchronize()
    assert rc == -1, (rc, _capi.last_error())      # B200_EINVAL
    assert _capi.launch_count() == before
    assert all(_untouched(buf) for buf, _ in bufs), "a rejected call wrote to a buffer"
