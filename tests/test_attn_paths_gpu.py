"""Every path of the attention dispatch (attn_paths.reachable: template instantiation x V path x epilogue x tiling)
against the fp64 reference, and the stream-ordered workspaces of split-KV and of the transpose pre-pass off the default
stream and inside CUDA graphs.

Each case of attn_paths.CASES is checked the way the sibling modules check their own:
  * outputs inside NaN guard bands (test_attn_numerics_gpu);
  * unsplit: attn_ref.o_bound / lse_bound of attn_mask_ref.reference on K/V expanded to H heads (attn_ref.rms_reference
    with the fused RMS norm); split: attn_split_ref.combine_bound; rows without a key exactly O = 0, lse = -inf;
  * GQA without a split bit for bit the same call on the expanded K/V; every non-RMS case again with lse=None, O bit
    for bit the same; _capi.launch_count() up by exactly the launches attn_paths.path restates;
  * the path itself on the device: under torch.profiler (in a child process) the recorded attn_fwd_kernel<...> is the
    restated instantiation, the transpose pre-pass runs exactly when the path has it, the combine exactly when it splits.
The largest |err| / bound per path is printed at the end of the module (pytest -s).
"""
import collections
import math

import pytest
import torch

import attn_mask_ref as M
import attn_paths as P
import attn_ref as R
import attn_split_ref as SR
from leetcuda_b200 import _capi, flash_attn, fused_ops
from test_attn_gqa_gpu import _inputs
from test_attn_numerics_gpu import RMS_G, _assert_margins, _guarded
from test_attn_seqlens_gpu import _kernels_per_call, profiled_names_of

pytestmark = pytest.mark.gpu

_ratios = collections.defaultdict(float)


def label(key):
    ds, bn, wg, vt, causal, gqa, split, prepass, rms, tiling = key
    flags = [f for f, on in (("vt", vt), ("causal", causal), ("gqa", gqa), ("split", split)) if on]
    return f"<{','.join([str(ds), str(bn), str(wg)] + flags)}> {'prepass' if prepass else '-'} {rms} {tiling}"


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    if _ratios:
        print("\nlargest |err| / bound per path (attn_ref.o_bound / lse_bound, rms_reference, "
              "attn_split_ref.combine_bound):")
        for key in sorted({k for k, _ in _ratios}):
            print(f"  {label(key):<48} O {_ratios[(key, 'O')]:.3f}  lse {_ratios[(key, 'lse')]:.3f}")


def _call(c, q, k, varg, o, lse):
    if c.rms:
        fused_ops.attn_rmsnorm(q, k, varg, o, RMS_G, v_transposed=c.vt, lse=lse)
    else:
        flash_attn.fmha_fwd(q, k, varg, o, v_transposed=c.vt, lse=lse, causal=c.causal, num_splits=c.splits)


def _run(c, q, k, varg):
    """O and lse in guarded buffers, and the launches the call counted."""
    obuf, o = _guarded(tuple(q.shape), torch.float16)
    lbuf, lse = _guarded(tuple(q.shape[:3]), torch.float32)
    torch.cuda.synchronize()
    n0 = _capi.launch_count()
    _call(c, q, k, varg, o, lse)
    launches = _capi.launch_count() - n0
    torch.cuda.synchronize()
    _assert_margins(obuf, "O")
    _assert_margins(lbuf, "lse")
    return o, lse, launches


def _check(key, got, want, bound, empty, what):
    """got within bound of want on the rows that see a key; empty rows exactly O = 0, lse = -inf."""
    for name, g, w, b in zip(("O", "lse"), got, want, bound):
        assert not bool(torch.isnan(g).any()), f"{what} {name}: NaN"
        if bool(empty.any()):
            assert bool((g[empty] == (-math.inf if name == "lse" else 0)).all()), f"{what} {name}: empty row"
        ne = ~empty
        err = (g.double()[ne] - w[ne]).abs()
        if err.numel() == 0:
            continue
        ratio = torch.nan_to_num(err / b[ne], nan=float("inf")).max().item()
        _ratios[(key, name)] = max(_ratios[(key, name)], ratio)
        if not bool((err <= b[ne]).all()):
            pytest.fail(f"{what} {name}: |err|/bound {ratio:.3g}")


@pytest.mark.parametrize("i", range(len(P.CASES_BY_SHAPE)), ids=lambda i: f"case{i}-D{P.CASES_BY_SHAPE[i].D}")
def test_path_against_fp64(i):
    c = P.CASES_BY_SHAPE[i]
    key, launches = P.path(c.B, c.H, c.Hkv, c.Nq, c.Nk, c.D, c.vt, c.causal, c.splits, c.rms)
    G, poly = c.H // c.Hkv, c.D <= 128
    sc = R.kernel_scale(c.D)
    for j, gen in enumerate(c.gens):
        what = f"{label(key)}: B{c.B} H{c.H} Hkv{c.Hkv} Nq{c.Nq} Nk{c.Nk} D{c.D} splits={c.splits} {gen}"
        q, k, v = _inputs(gen, c.B, c.H, c.Hkv, c.Nq, c.Nk, c.D, None, seed=7919 * i + j)
        varg = v.transpose(-2, -1).contiguous() if c.vt else v
        o, lse, n = _run(c, q, k, varg)
        assert n == launches, f"{what}: {n} launches, the path has {launches}"
        exact = M.exact_scores(gen)
        if c.splits > 1:
            parts = SR.part_references(q, k, v, sc, c.causal, c.splits, exact)
            want_o, want_l, empty, ob, lb = SR.combine_bound(parts, poly)
        else:
            ref = M.reference(q, SR.expand(k, G), SR.expand(v, G), sc, c.causal, exact_scores=exact)
            pre, ob = R.o_bound(ref, poly)
            want_o, want_l, empty, lb = ref["o"], ref["lse"], ref["empty"], R.lse_bound(ref, poly)
            if c.rms:
                want_o, ob = R.rms_reference(ref, RMS_G, pre)
        _check(key, (o, lse), (want_o, want_l), (ob, lb), empty, what)

        if G > 1 and c.splits == 1:
            ke, ve = SR.expand(k, G).contiguous(), SR.expand(v, G).contiguous()
            eo, el, _ = _run(c, q, ke, ve.transpose(-2, -1).contiguous() if c.vt else ve)
            assert torch.equal(o, eo) and torch.equal(lse, el), what + ": not bitwise the expanded-K/V call"
        if not c.rms:
            o2 = torch.empty_like(o)
            _call(c, q, k, varg, o2, None)
            torch.cuda.synchronize()
            assert torch.equal(o, o2), what + ": O with lse=None differs"


# torch.profiler runs in a child process, all cases in one session (test_attn_seqlens_gpu._kernels_per_call); this
# process never starts it.
def _profile_all_cases():
    """Child process: the CUDA kernel names of every case, as one JSON line on stdout."""
    import json
    fns = []
    for i, c in enumerate(P.CASES_BY_SHAPE):
        q, k, v = _inputs("randn", c.B, c.H, c.Hkv, c.Nq, c.Nk, c.D, None, seed=i)
        varg = v.transpose(-2, -1).contiguous() if c.vt else v
        o, lse = torch.empty_like(q), torch.empty(q.shape[:3], device="cuda")
        fns.append(lambda a=(c, q, k, varg, o, lse): _call(*a))
    print("KERNEL_NAMES " + json.dumps(_kernels_per_call(fns)))


@pytest.fixture(scope="module")
def profiled_names():
    return profiled_names_of("test_attn_paths_gpu")


@pytest.mark.parametrize("i", range(len(P.CASES_BY_SHAPE)), ids=lambda i: f"case{i}-D{P.CASES_BY_SHAPE[i].D}")
def test_kernel_names(profiled_names, i):
    c = P.CASES_BY_SHAPE[i]
    key, _ = P.path(c.B, c.H, c.Hkv, c.Nq, c.Nk, c.D, c.vt, c.causal, c.splits, c.rms)
    what = f"{label(key)}: B{c.B} H{c.H} Hkv{c.Hkv} Nq{c.Nq} Nk{c.Nk} D{c.D} splits={c.splits}"
    names = profiled_names[i] if i < len(profiled_names) else []
    assert names, what + ": the profiler recorded no kernel"
    assert P.parse_instantiations(names) == [P.instantiation(key)], f"{what}: ran {names}"
    assert sum("transpose_dn_to_nd_kernel" in s for s in names) == int(key[7]), f"{what}: ran {names}"
    assert sum("attn_combine_kernel" in s for s in names) == int(key[6]), f"{what}: ran {names}"


# ------------------------------------------------------------------ workspaces under streams and graphs
# (B, H, Hkv, Nq, Nk, D, vt, causal, splits): a D = 128 decode split; a split of the D <= 64 vt kernel; a causal
# split behind the transpose pre-pass, which holds both stream-ordered workspaces at once.
STREAM_PATHS = [(1, 8, 2, 1, 1000, 128, False, False, 4),
                (1, 8, 2, 5, 776, 64, True, False, 5),
                (1, 4, 2, 130, 776, 264, True, True, 3)]


def _fresh(B, H, Hkv, Nq, Nk, D, vt, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    q = torch.randn(B, H, Nq, D, device="cuda", dtype=torch.half, generator=g)
    k = torch.randn(B, Hkv, Nk, D, device="cuda", dtype=torch.half, generator=g)
    v = torch.randn(B, Hkv, *((D, Nk) if vt else (Nk, D)), device="cuda", dtype=torch.half, generator=g)
    return q, k, v


def _into(q, k, v, o, lse, vt, causal, splits):
    flash_attn.fmha_fwd(q, k, v, o, v_transposed=vt, lse=lse, causal=causal, num_splits=splits)


def _eager(q, k, v, vt, causal, splits):
    o, lse = torch.empty_like(q), torch.empty(q.shape[:3], device="cuda")
    _into(q, k, v, o, lse, vt, causal, splits)
    torch.cuda.synchronize()
    return o, lse


@pytest.mark.parametrize("shape", STREAM_PATHS, ids=["decode-D128", "vt-D64", "prepass-causal-D264"])
def test_workspaces_on_a_side_stream_and_in_a_graph(shape):
    B, H, Hkv, Nq, Nk, D, vt, causal, splits = shape
    assert P.path(B, H, Hkv, Nq, Nk, D, vt, causal, splits, False)[0][6]

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        q, k, v = _fresh(B, H, Hkv, Nq, Nk, D, vt, seed=1)
        o, lse = torch.empty_like(q), torch.empty(q.shape[:3], device="cuda")
        _into(q, k, v, o, lse, vt, causal, splits)
    side.synchronize()
    want = _eager(q, k, v, vt, causal, splits)
    assert torch.equal(o, want[0]) and torch.equal(lse, want[1]), "side stream"

    sq, sk, sv = (torch.zeros_like(x) for x in (q, k, v))
    so, sl = torch.empty_like(q), torch.empty(q.shape[:3], device="cuda")
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            _into(sq, sk, sv, so, sl, vt, causal, splits)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        _into(sq, sk, sv, so, sl, vt, causal, splits)
    for rep in range(2):
        q, k, v = _fresh(B, H, Hkv, Nq, Nk, D, vt, seed=10 + rep)
        for s, x in ((sq, q), (sk, k), (sv, v)):
            s.copy_(x)
        graph.replay()
        torch.cuda.synchronize()
        want = _eager(q, k, v, vt, causal, splits)
        assert torch.equal(so, want[0]) and torch.equal(sl, want[1]), f"graph replay {rep}"


@pytest.mark.parametrize("shape", STREAM_PATHS, ids=["decode-D128", "vt-D64", "prepass-causal-D264"])
def test_workspaces_of_two_streams_at_once(shape):
    """Two calls with different workspace sizes (Nk and the split count differ) on two streams, not synchronised
    with each other: each is bit for bit its serial result."""
    B, H, Hkv, Nq, Nk, D, vt, causal, splits = shape
    calls = [(Nk, splits), (Nk - 256, splits + 2)]
    inputs = [_fresh(B, H, Hkv, Nq, n, D, vt, seed=20 + j) for j, (n, _) in enumerate(calls)]
    serial = [_eager(*x, vt, causal, s) for x, (_, s) in zip(inputs, calls)]
    outs = [(torch.empty_like(x[0]), torch.empty(x[0].shape[:3], device="cuda")) for x in inputs]
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    torch.cuda.synchronize()
    for st, x, (o, lse), (_, s) in zip(streams, inputs, outs, calls):
        with torch.cuda.stream(st):
            _into(*x, o, lse, vt, causal, s)
    torch.cuda.synchronize()
    for j in range(2):
        assert torch.equal(outs[j][0], serial[j][0]) and torch.equal(outs[j][1], serial[j][1]), f"call {j}"
