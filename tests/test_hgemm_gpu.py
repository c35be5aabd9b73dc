"""GPU parity tests of the HGEMM path: every call goes through the C ABI
(leetcuda_b200.hgemm -> ctypes -> b200_hgemm_f16).  The checker is the CPU oracle
(oracle/oracle.c) on small seeded inputs, the committed golden outputs of the
reference's own kernels, and size-independent properties at the BASELINE sizes.

Tolerance (north_star): fp16 rtol=1e-2 / atol=1e-2 against the fp32-accumulated
oracle.  Integer-valued inputs are checked BIT-EXACTLY.
"""
import math

import numpy as np
import pytest
import torch

import gemm_ref
from leetcuda_b200 import _capi, hgemm
from oracle import oracle as O
from oracle.gen_golden import HGEMM_CASES, hgemm_inputs

pytestmark = pytest.mark.gpu
RTOL = ATOL = 1e-2


def _dev(x):
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def _as_col_major(b):  # reference tools/utils.py:151-156
    return b.t().reshape(b.shape).contiguous()


SENT16 = 0x7E5B      # a NaN bit pattern the GEMM never produces
MARGIN = 256         # elements of C's guard bands (512 B: the alignment of C is kept)


def _guarded_c(M, N):
    """C as a view inside a larger buffer filled with SENT16: (buffer, C)."""
    buf = torch.empty(M * N + 2 * MARGIN, dtype=torch.half, device="cuda")
    buf.view(torch.int16).fill_(SENT16)
    return buf, buf[MARGIN:MARGIN + M * N].view(M, N)


def _untouched(t):
    return bool((t.view(torch.int16) == SENT16).all())


def _run(a, b, tn=False, op=None):
    M, K = a.shape
    N = b.shape[1]
    c = torch.full((M, N), float("nan"), dtype=torch.half, device="cuda")
    if op is None:
        hgemm.hgemm(a, _as_col_major(b) if tn else b, c, tn=tn)
    else:
        args = (a, _as_col_major(b) if tn else b, c)
        if "stages" in op.__doc__:
            op(*args, 2, False, 1)
        else:
            op(*args)
    torch.cuda.synchronize()
    return c


@pytest.mark.parametrize("tn", [False, True])
@pytest.mark.parametrize("shape", [(128, 128, 64), (256, 256, 128), (512, 512, 512),
                                   (384, 640, 200), (136, 264, 72), (8, 8, 8), (1000, 24, 4096),
                                   (128, 24, 512), (128, 64, 512), (1000, 72, 512), (2600, 2000, 136)])
def test_vs_oracle_small(shape, tn):
    """configs[0] (512^3) and ragged shapes the reference cannot run, vs the CPU oracle, with guard bands around C.

    2600 x 2000 x 136 reaches the partial raster group and the persistent loop: on 132 SMs the host scores 336 tiles of
    128 x 128 (3 waves, 0.9 x 336 / 396 = 0.76) against 168 of 128 x 256 (2 waves, 168 / 264 = 0.64), so it runs on
    the 128-column tile, 2-3 tiles per CTA; tiles_m = 21 is a group of 16 m-tiles and then a partial group of 5,
    which, being odd, walks the n-tiles backwards.  M, N and K are all ragged."""
    M, N, K = shape
    a_np, b_np = hgemm_inputs(M, N, K, seed=M + N + K)
    want = O.hgemm_f32acc(a_np, b_np).astype(np.float32)
    a, b = _dev(a_np), _dev(b_np)
    buf, c = _guarded_c(M, N)
    hgemm.hgemm(a, _as_col_major(b) if tn else b, c, tn=tn)
    torch.cuda.synchronize()
    assert _untouched(buf[:MARGIN]) and _untouched(buf[-MARGIN:]), "store outside C"
    got = c.cpu().numpy().astype(np.float32)
    np.testing.assert_allclose(got, want, rtol=RTOL, atol=ATOL)
    # and tighter than the tolerance requires: fp32 accumulation differs from the oracle only by
    # summation order, so at most one fp16 ulp of the result
    truth = O.hgemm_f64(a_np, b_np)
    ulp = np.maximum(np.abs(truth), 1.0) * 2.0 ** -10
    assert np.all(np.abs(got - truth) <= 1.01 * ulp)
    # and element by element within the bound derived in gemm_ref.py
    ref = gemm_ref.reference(a_np, b_np, "f16")
    assert np.all(np.abs(got - ref["c"]) <= gemm_ref.bound(ref))


def test_every_op_name_computes_the_same_gemm():
    """The whole op surface (36 GEMM names) is callable and agrees with the oracle."""
    M, N, K = 256, 256, 128
    a_np, b_np = hgemm_inputs(M, N, K, seed=5)
    want = O.hgemm_f32acc(a_np, b_np).astype(np.float32)
    a, b = _dev(a_np), _dev(b_np)
    before = _capi.launch_count()
    n_ours = 0
    for name in hgemm.OP_NAMES:
        op = getattr(hgemm, name)
        tn = name.endswith("_tn") or "_tn_" in name
        got = _run(a, b, tn=tn, op=op).cpu().numpy().astype(np.float32)
        np.testing.assert_allclose(got, want, rtol=RTOL, atol=ATOL, err_msg=name)
        n_ours += 0 if "cublas" in name else 1
    assert _capi.launch_count() - before == n_ours  # every non-cuBLAS op launched OUR kernel


@pytest.mark.parametrize("case", HGEMM_CASES)
def test_vs_reference_golden(case):
    """Against outputs of the reference's own kernels, recorded once and stored in tests/golden."""
    from pathlib import Path
    M, N, K, seed = case
    f = Path(__file__).parent / "golden" / f"hgemm_{M}x{N}x{K}_s{seed}.npz"
    if not f.exists():
        pytest.skip("golden file not generated yet")
    import json
    g = np.load(f)
    sub = json.loads(str(g["meta"])).get("subsample", 1)
    a_np, b_np = hgemm_inputs(M, N, K, seed)
    truth = O.hgemm_f64(a_np, b_np)[::sub, ::sub]
    got = _run(_dev(a_np), _dev(b_np)).cpu().numpy().astype(np.float64)[::sub, ::sub]
    ours_err = np.abs(got - truth).max()
    for name in g.files:
        if name == "meta":
            continue
        ref = g[name].astype(np.float64)
        ref_err = np.abs(ref - truth).max()
        # gate of SURVEY §8c: error vs truth no worse than the reference's own kernels
        assert ours_err <= ref_err + 1e-6, (name, ours_err, ref_err)
        # and element-wise agreement with the reference within the K-scaled fp16-accumulation band
        np.testing.assert_allclose(got, ref, rtol=RTOL, atol=ATOL * max(1.0, K / 64), err_msg=name)


@pytest.mark.parametrize("case", HGEMM_CASES)
def test_acc_f16_mode_reproduces_reference_bits(case):
    """Parity mode (wgmma D format f16): the reference's fp16-accumulating kernels are reproduced
    bit for bit on >= 99 % of the outputs, the rest within one fp16 ulp at the output magnitude —
    the same agreement the reference's own kernels have with the k16-chunked oracle."""
    import json
    from pathlib import Path
    M, N, K, seed = case
    f = Path(__file__).parent / "golden" / f"hgemm_{M}x{N}x{K}_s{seed}.npz"
    if not f.exists():
        pytest.skip("golden file not generated yet")
    g = np.load(f)
    sub = json.loads(str(g["meta"])).get("subsample", 1)
    a_np, b_np = hgemm_inputs(M, N, K, seed)
    a, b = _dev(a_np), _dev(b_np)
    c = torch.empty(M, N, dtype=torch.half, device="cuda")
    hgemm.hgemm(a, b, c, acc="f16")
    torch.cuda.synchronize()
    got = c.cpu().numpy()[::sub, ::sub]
    o16 = O.hgemm_f16acc(a_np, b_np, k_chunk=16)[::sub, ::sub]
    ulp = 2.0 ** (np.floor(np.log2(np.abs(o16.astype(np.float64)).max())) - 10)
    assert np.mean(got == o16) >= 0.99, np.mean(got == o16)
    assert np.abs(got.astype(np.float64) - o16.astype(np.float64)).max() <= ulp
    ref = g["hgemm_mma_m16n8k16_mma2x4_warp4x4x2_stages_dsmem_swizzle"]
    assert np.mean(got == ref) >= 0.99, np.mean(got == ref)
    # TN layout, same mode, same bits
    c2 = torch.empty(M, N, dtype=torch.half, device="cuda")
    hgemm.hgemm(a, _as_col_major(b), c2, tn=True, acc="f16")
    torch.cuda.synchronize()
    assert torch.equal(c, c2)


def test_acc_f16_mode_vs_reference_kernel_at_headline_size():
    """BASELINE configs[1] (8192^3, randn inputs): the fp16-accumulate parity mode against the reference's arithmetic at
    the headline size.  The reference's kernels round the accumulator to fp16 after every k16 MMA in ascending k order;
    oracle_hgemm_f16acc(k_chunk=16) restates that on the CPU and reproduces the reference kernels' recorded outputs bit
    for bit (tests/test_oracle_golden.py).  Against it, on 32 rows spread over all row tiles, the outputs must be
    bit-identical on >= 98 % (measured on H100: 98.5 % — the wgmma f16 accumulator rounds once per k16 instruction
    like the restatement, but over 512 roundings an occasional tie resolves differently) and within 2 fp16 ulps of the
    largest output elsewhere.  Where the reference's flagship
    kernel (hgemm_mma_m16n8k16_mma2x4_warp4x4x2_stages_dsmem_swizzle) has been built into oracle/_ref, the same holds
    against it on all 67 M outputs.  (The default fp32-accumulate mode cannot be held to allclose(1e-2) against an
    fp16-accumulating kernel at K = 8192 — SURVEY §7 hard part 1 — which is why this mode exists.)"""
    from oracle.build_ref import load_prebuilt
    S = 8192
    g = torch.Generator(device="cuda").manual_seed(8192)
    a = torch.randn(S, S, device="cuda", dtype=torch.half, generator=g)
    b = torch.randn(S, S, device="cuda", dtype=torch.half, generator=g)
    c = torch.zeros(S, S, device="cuda", dtype=torch.half)
    hgemm.hgemm(a, b, c, acc="f16")
    torch.cuda.synchronize()
    rows = torch.arange(0, S, S // 32, device="cuda")
    o16 = O.hgemm_f16acc(a[rows].cpu().numpy(), b.cpu().numpy(), k_chunk=16)
    got = c[rows].cpu().numpy()
    assert np.mean(got == o16) >= 0.98, np.mean(got == o16)
    ulp = 2.0 ** (math.floor(math.log2(np.abs(o16.astype(np.float64)).max())) - 10)
    assert np.abs(got.astype(np.float64) - o16.astype(np.float64)).max() <= 2 * ulp
    ref = load_prebuilt("ref_hgemm")
    if ref is not None:
        c_ref = torch.zeros(S, S, device="cuda", dtype=torch.half)
        ref.hgemm_mma_m16n8k16_mma2x4_warp4x4x2_stages_dsmem_swizzle(a, b, c_ref, 2, True, 2048)
        torch.cuda.synchronize()
        same = (c == c_ref).float().mean().item()
        assert same >= 0.99, same
        ulp = 2.0 ** (math.floor(math.log2(c_ref.float().abs().max().item())) - 10)
        assert (c.float() - c_ref.float()).abs().max().item() <= 2 * ulp
    # and the default mode is the more accurate of the two against an fp32 product of the same operands
    c32 = torch.zeros(S, S, device="cuda", dtype=torch.half)
    hgemm.hgemm(a, b, c32)
    rows = slice(0, 1024)
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    truth = a[rows].float() @ b.float()
    torch.backends.cuda.matmul.allow_tf32 = prev
    err32 = (c32[rows].float() - truth).abs().max().item()
    err16 = (c[rows].float() - truth).abs().max().item()
    assert err32 < err16, (err32, err16)


@pytest.mark.parametrize("tn", [False, True])
def test_bit_exact_integer_inputs_full_size(tn):
    """BASELINE configs[1] (8192^3): ternary inputs make every partial sum an exactly
    representable integer, so the result must equal the integer product bit for bit."""
    S = 8192
    g = torch.Generator(device="cuda").manual_seed(1)
    a = torch.randint(-1, 2, (S, S), device="cuda", generator=g).half()
    b = torch.randint(-1, 2, (S, S), device="cuda", generator=g).half()
    want = (a.float() @ b.float())  # exact in fp32 (|sum| << 2^24)
    assert want.abs().max().item() < 2048  # exactly representable in fp16
    got = _run(a, b, tn=tn)
    assert torch.equal(got.float(), want)


def test_identity_and_linearity_full_size():
    S = 8192
    g = torch.Generator(device="cuda").manual_seed(2)
    a = torch.randn(S, S, device="cuda", dtype=torch.half, generator=g)
    eye = torch.eye(S, device="cuda", dtype=torch.half)
    assert torch.equal(_run(a, eye), a)                      # A @ I == A, bit exact
    b = torch.randn(S, 256, device="cuda", dtype=torch.half, generator=g)
    c1 = _run(a, b)
    c2 = _run(a, (b * 2).contiguous())
    # exact power-of-two scaling wherever the fp16 result is normal; a subnormal result is rounded on the fixed
    # 2^-24 grid, so there doubling before or after the rounding may differ by that one step
    normal = c2.float().abs() >= 2.0 ** -14
    assert torch.equal(c2[normal], (c1 * 2)[normal])
    assert ((c2.float() - c1.float() * 2).abs() <= 2.0 ** -24).all()
    assert torch.equal(_run(a, b, tn=True), c1)              # NN and TN agree bit for bit


def test_tile_widths_agree():
    """The 128- and 256-column tiles compute the same bits.  The host picks the 128-column tile when its share of busy
    SMs in the last wave, times 0.9, beats that of the 256-column tile.  On 132 SMs the 4096 x 4096 product has 512
    tiles of 128 x 256 (4 waves, 512 / 528 = 0.97) against 1024 of 128 x 128 (8 waves, 0.9 x 1024 / 1056 = 0.87), so it
    runs on the 256-column tile; a 256-row shard of it has 32 tiles of 128 x 256 (32 / 132 = 0.24) against 64 of
    128 x 128 (0.9 x 64 / 132 = 0.44) and runs on the 128-column tile."""
    if torch.cuda.get_device_properties(0).multi_processor_count != 132:
        pytest.skip("the tile choices in the docstring are worked out for 132 SMs")
    M, N, K = 4096, 4096, 2048
    a_np, b_np = hgemm_inputs(M, N, K, seed=9)
    a, b = _dev(a_np), _dev(b_np)
    full = _run(a, b)
    row0, rows = 1024, 256
    buf, c = _guarded_c(M, N)
    rc = _capi.lib().b200_hgemm_f16_rows(a[row0:row0 + rows].data_ptr(), b.data_ptr(), c.data_ptr(), rows, N, K,
                                         _capi.B_ROW_MAJOR_KN, row0, torch.cuda.current_stream().cuda_stream)
    assert rc == 0, _capi.last_error()
    torch.cuda.synchronize()
    assert torch.equal(c[row0:row0 + rows], full[row0:row0 + rows])
    # the shard call writes its own rows of C and nothing else
    assert _untouched(buf[:MARGIN + row0 * N]) and _untouched(buf[MARGIN + (row0 + rows) * N:])


def test_row_shard_entry_point_matches_full():
    """b200_hgemm_f16_rows (the multi-GPU shard call) reproduces the full product."""
    M, N, K = 1024, 512, 768
    a_np, b_np = hgemm_inputs(M, N, K, seed=3)
    a, b = _dev(a_np), _dev(b_np)
    full = _run(a, b)
    c = torch.zeros(M, N, dtype=torch.half, device="cuda")
    lib = _capi.lib()
    for r in range(4):
        rows = M // 4
        rc = lib.b200_hgemm_f16_rows(a[r * rows:(r + 1) * rows].data_ptr(), b.data_ptr(), c.data_ptr(),
                                     rows, N, K, 0, r * rows, torch.cuda.current_stream().cuda_stream)
        assert rc == 0, _capi.last_error()
    torch.cuda.synchronize()
    assert torch.equal(c, full)


def test_host_buffer_entry_point():
    M, N, K = 256, 384, 512
    a_np, b_np = hgemm_inputs(M, N, K, seed=4)
    c_np = np.zeros((M, N), np.float16)
    rc = _capi.lib().b200_hgemm_f16_host(a_np.ctypes.data, b_np.ctypes.data, c_np.ctypes.data, M, N, K, 0, None)
    assert rc == 0, _capi.last_error()
    np.testing.assert_allclose(c_np.astype(np.float32), O.hgemm_f32acc(a_np, b_np).astype(np.float32),
                               rtol=RTOL, atol=ATOL)


def test_host_buffer_entry_point_pipelined_panels():
    """M > 1024 rows: the host entry pipelines several row panels through the copy engines."""
    M, N, K = 2600, 256, 512
    a_np, b_np = hgemm_inputs(M, N, K, seed=6)
    a, b = torch.from_numpy(a_np).pin_memory(), torch.from_numpy(b_np).pin_memory()
    c = torch.zeros(M, N, dtype=torch.half).pin_memory()
    for _ in range(2):   # second call re-uses the cached workspace, streams and events
        c.zero_()
        hgemm.hgemm_host(a, b, c)
        np.testing.assert_allclose(c.numpy().astype(np.float32), O.hgemm_f32acc(a_np, b_np).astype(np.float32),
                                   rtol=RTOL, atol=ATOL)
    with pytest.raises(RuntimeError, match="host tensors"):
        hgemm.hgemm_host(a.cuda(), b, c)


def test_bad_alignment_is_an_error_not_a_crash():
    a = torch.zeros(128, 64, dtype=torch.half, device="cuda")
    b = torch.zeros(64, 132, dtype=torch.half, device="cuda")   # N % 8 != 0
    c = torch.zeros(128, 132, dtype=torch.half, device="cuda")
    with pytest.raises(RuntimeError, match="multiples of 8"):
        hgemm.hgemm(a, b, c)
