"""fp8 (e4m3) scaled GEMM on the GPU (hgemm.scaled_mm -> b200_gemm_e4m3) against the fp64 reference and per-element bound
of gemm_fp8_ref.py: every recipe x output type over the shape table, NaN guard bands around C, inputs and scales left
unchanged, one launch per call, CUDA-graph replay with new scale values, a C past 2^31 elements, 8192^3, and
torch._scaled_mm on the same inputs within the same bound."""
import pytest
import torch

import gemm_fp8_ref as R
from leetcuda_b200 import _capi, hgemm

pytestmark = pytest.mark.gpu
DEV = "cuda"
GUARD = 64                                        # elements on either side of C (16-byte aligned)
_worst = {}


def _dev(inputs, scales):
    """Inputs (a, b_nk, info) and scales on the GPU; b as the [K,N] column-major view of the [N,K] rows."""
    (a, b, _), (sa, sb) = inputs, scales
    return a.to(DEV), b.to(DEV).t(), sa.to(DEV), sb.to(DEV)


def _guarded_c(M, N, od):
    buf = torch.full((M * N + 2 * GUARD,), float("nan"), dtype=od, device=DEV)
    return buf, buf[GUARD:GUARD + M * N].view(M, N)


def _run(a, b, sa, sb, recipe, od, c=None):
    buf = None
    if c is None:
        buf, c = _guarded_c(a.shape[0], b.shape[1], od)
    keep = [x.clone() for x in (a, b, sa, sb)]
    n0 = _capi.launch_count()
    hgemm.scaled_mm(a, b, c, sa, sb, scale_recipe=recipe)
    torch.cuda.synchronize()
    assert _capi.launch_count() == n0 + 1
    for x, y in zip((a, b, sa, sb), keep):
        assert torch.equal(x.view(torch.uint8) if x.dtype == R.E4 else x, y.view(torch.uint8) if y.dtype == R.E4 else y)
    if buf is not None:
        assert buf[:GUARD].isnan().all() and buf[-GUARD:].isnan().all()
    return c


def _check(c, ref, od, gen, tag):
    got = c.double()[ref["rows"]] if ref["rows"] is not None else c.double()
    bd = R.bound(ref, od)
    assert torch.isfinite(got).all(), tag
    ratio = ((got - ref["c"]).abs() / bd).max().item()
    key = (tag, gen)
    _worst[key] = max(_worst.get(key, 0.0), ratio)
    assert ratio <= 1.0, (tag, gen, ratio)
    if gen in R.EXACT:
        assert torch.equal(c[ref["rows"]], R.rounded(ref, od)), (tag, gen)


@pytest.mark.parametrize("shape", R.SHAPES, ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("od", R.OUT_DTYPES, ids=lambda d: str(d)[6:])
@pytest.mark.parametrize("recipe", R.RECIPES)
def test_shape_matrix(recipe, od, shape):
    M, N, K = shape
    gens = ("randn", "int", "k_probe") if M * N * K <= 2 ** 28 else ("randn", "int")
    for i, gen in enumerate(gens):
        a, b, sa, sb = _dev(R.make_inputs(gen, M, N, K, seed=i), R.make_scales(recipe, M, N, K, gen in R.EXACT, i))
        c = _run(a, b, sa, sb, recipe, od)
        _check(c, R.reference(a, b.t(), sa, sb, recipe), od, gen, f"{recipe}-{str(od)[6:]}")


@pytest.mark.parametrize("gen", ["binade", "cancel", "a_probe"])
@pytest.mark.parametrize("recipe", R.RECIPES)
def test_other_generators(recipe, gen):
    M, N, K = 385, 520, 2048
    for od in R.OUT_DTYPES:
        a, b, sa, sb = _dev(R.make_inputs(gen, M, N, K, seed=5), R.make_scales(recipe, M, N, K, gen in R.EXACT, 5))
        c = _run(a, b, sa, sb, recipe, od)
        _check(c, R.reference(a, b.t(), sa, sb, recipe), od, gen, f"{recipe}-{str(od)[6:]}")


def test_kernel_name_under_profiler():
    M, N, K = 256, 256, 256
    a, b, sa, sb = _dev(R.make_inputs("randn", M, N, K), R.make_scales("block", M, N, K, False))
    c = torch.empty(M, N, dtype=torch.bfloat16, device=DEV)
    hgemm.scaled_mm(a, b, c, sa, sb, scale_recipe="block")
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        hgemm.scaled_mm(a, b, c, sa, sb, scale_recipe="block")
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if "gemm_e4m3_kernel" in e.name]
    assert names and all("bfloat16" in n for n in names), [e.name for e in prof.events()][:20]


@pytest.mark.parametrize("recipe", R.RECIPES)
def test_graph_replay_with_new_scales(recipe):
    M, N, K = 300, 264, 384
    a, b, sa, sb = _dev(R.make_inputs("int", M, N, K, seed=9), R.make_scales(recipe, M, N, K, True, 9))
    c = torch.empty(M, N, dtype=torch.float16, device=DEV)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        hgemm.scaled_mm(a, b, c, sa, sb, scale_recipe=recipe)      # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        hgemm.scaled_mm(a, b, c, sa, sb, scale_recipe=recipe)
    for seed in (11, 12):
        na, nb = R.make_scales(recipe, M, N, K, True, seed)
        sa.copy_(na.to(DEV))
        sb.copy_(nb.to(DEV))
        c.fill_(float("nan"))
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(c, R.rounded(R.reference(a, b.t(), sa, sb, recipe), torch.float16))


def _free_gib():
    return torch.cuda.mem_get_info()[0] / 2 ** 30


def test_c_past_2_31_elements():
    M, N, K = 33000, 65536, 128                   # C: 2,162,688,000 elements (4.0 GiB)
    if _free_gib() < 8:
        pytest.skip(f"needs 8 GiB free, {_free_gib():.1f} GiB")
    assert M * N > 2 ** 31
    a, b, sa, sb = _dev(R.make_inputs("int", M, N, K, seed=4), R.make_scales("row", M, N, K, True, 4))
    c = torch.full((M, N), float("nan"), dtype=torch.bfloat16, device=DEV)
    n0 = _capi.launch_count()
    hgemm.scaled_mm(a, b, c, sa, sb, scale_recipe="row")
    torch.cuda.synchronize()
    assert _capi.launch_count() == n0 + 1
    rows = [0, 2 ** 31 // N - 1, 2 ** 31 // N, M - 1]
    ref = R.reference(a, b.t(), sa, sb, "row", rows=rows)
    _check(c, ref, torch.bfloat16, "int", "row-bfloat16-2^31")
    del c


@pytest.mark.parametrize("recipe", R.RECIPES)
def test_8192_cubed_sampled_rows(recipe):
    M = N = K = 8192
    a, b, sa, sb = _dev(R.make_inputs("randn", M, N, K, seed=8), R.make_scales(recipe, M, N, K, False, 8))
    c = _run(a, b, sa, sb, recipe, torch.bfloat16)
    rows = [0, 1, 127, 128, 4095, 4096, 8190, 8191]
    _check(c, R.reference(a, b.t(), sa, sb, recipe, rows=rows), torch.bfloat16, "randn", f"{recipe}-8192^3")


def _torch_scaled_mm(a, b, sa, sb, recipe, od, fast):
    """torch._scaled_mm with this recipe's scales in torch's layout, or a skip reason."""
    M, N = a.shape[0], b.shape[1]
    try:
        if recipe == "tensor":
            return torch._scaled_mm(a, b, sa.reshape(()), sb.reshape(()), out_dtype=od, use_fast_accum=fast), None
        if recipe == "row":
            return torch._scaled_mm(a, b, sa.reshape(M, 1), sb.reshape(1, N), out_dtype=od,
                                    use_fast_accum=fast), None
        return torch._scaled_mm(a, b, sa, sb.t(), out_dtype=od, use_fast_accum=fast), None
    except (RuntimeError, TypeError, NotImplementedError) as e:
        return None, f"torch._scaled_mm does not take {recipe} scaling with {od} here: {str(e).splitlines()[0][:200]}"


@pytest.mark.parametrize("gen", ["randn", "binade", "cancel"])
@pytest.mark.parametrize("recipe", R.RECIPES)
def test_against_torch_scaled_mm(recipe, gen):
    M, N, K = 1024, 1536, 4096
    od = torch.bfloat16
    a, b, sa, sb = _dev(R.make_inputs(gen, M, N, K, seed=6), R.make_scales(recipe, M, N, K, False, 6))
    ours = _run(a, b, sa, sb, recipe, od)
    ref = R.reference(a, b.t(), sa, sb, recipe)
    theirs, why = _torch_scaled_mm(a, b, sa, sb, recipe, od, fast=False)
    bd = R.bound(ref, od)
    r_ours = ((ours.double() - ref["c"]).abs() / bd).max().item()
    print(f"\n[fp8 gemm] {recipe:6s} {gen:6s} max |err|/bound: ours {r_ours:.4f}", end="")
    assert r_ours <= 1.0
    if theirs is None:
        pytest.skip(why)
    r_torch = ((theirs.double() - ref["c"]).abs() / bd).max().item()
    print(f"  torch._scaled_mm {r_torch:.4f}", end="")
    assert r_torch <= 1.0, r_torch


def test_zz_print_worst_ratios():
    for (tag, gen), r in sorted(_worst.items()):
        print(f"[fp8 gemm] max |err|/bound {tag:22s} {gen:8s} {r:.4f}")
