"""Packed variable-length attention (flash_attn.fmha_varlen_fwd, b200_fmha_fwd_{f16,bf16}_varlen[_paged]) on the GPU,
over every instantiation of attn_varlen_ref.CASES_BY_SHAPE.

Every case builds padded inputs (test_attn_gqa_gpu._inputs), packs them token-major with the raw lengths of the row
(a sequence longer than max_seqlen keeps its extra rows in the packed tensors) and poisons what no sequence may read or
write: Q rows past a sequence's Lq_b and past cu_q[B] hold NaN; K / V rows past Lk_b and past cu_k[B] hold NaN, +-Inf
or 65504 (unused pool pages too, paged); with randn inputs the first kBN keys of sequence b+1 are aimed at sequence
b's queries (large scores, V = 100), so a leak through b's last partial key block exceeds the bound.  O and lse sit in
NaN guard bands and are sentinel-filled; the rows no sequence owns must come back unchanged.  Checked:
  * bit for bit fmha_fwd(seqlens_q=, seqlens_k=, num_splits=1) (paged: with block_table=) on the padded copies;
  * the fp64 reference with each sequence's visibility (attn_seqlens_ref.reference; attn_ref / attn_bf16_ref bounds);
    rows without a visible key exactly O = 0 and lse = -inf; the inputs come back unchanged;
  * _capi.launch_count() up by exactly 1; under torch.profiler (in a child process) the restated kernel name and no
    device-to-host copy.
Then CUDA graphs replayed with new offsets, lengths and tables, a side stream, chunked prefill merged through
merge_attn_states, and every shape of tools/bench_attn_varlen.py at full size.  The largest |err| / bound per path is
printed at the end of the module (pytest -s).
"""
import collections
import importlib.util
import math
import time
from pathlib import Path

import numpy as np
import pytest
import torch

import attn_bf16_ref as BF
import attn_mask_ref as M
import attn_ref as R
import attn_seqlens_ref as S
import attn_split_ref as SR
import attn_varlen_ref as V
import merge_ref as MR
from leetcuda_b200 import _capi, flash_attn
from leetcuda_b200 import merge_attn_states as MA
from test_attn_gqa_gpu import _inputs
from test_attn_numerics_gpu import MARGIN
from test_attn_paged_gpu import paginate
from test_attn_seqlens_gpu import _kernels_per_call, _lens, _poison, profiled_names_of

pytestmark = pytest.mark.gpu

_ratios = collections.defaultdict(float)
_POISON = (float("nan"), float("inf"), float("-inf"), 65504.0)
_DT = {"fp16": torch.float16, "bf16": torch.bfloat16}
_SENT = {torch.float16: 0x7E01, torch.bfloat16: 0x7FC1, torch.float32: 0x7FC00001}   # NaN payloads no store makes
_BITS = {torch.float16: torch.int16, torch.bfloat16: torch.int16, torch.float32: torch.int32}


def label(key):
    if key[0] == "merge":
        return f"merge_attn_states {key[1]}"
    ds, bn, wg, causal, paged, t = key
    flags = [f for f, on in (("causal", causal), ("paged", paged)) if on]
    return f"<{','.join([str(ds), str(bn), str(wg)] + flags + [t])}>"


@pytest.fixture(scope="module", autouse=True)
def _report():
    t0 = time.time()
    yield
    if _ratios:
        print("\nlargest |err| / bound per path (attn_ref / attn_bf16_ref o_bound, lse_bound):")
        for key in sorted({k for k, _ in _ratios}, key=str):
            print(f"  {label(key):<48} O {_ratios[(key, 'O')]:.3f}  lse {_ratios[(key, 'lse')]:.3f}")
    print(f"module time {time.time() - t0:.1f} s")


# ------------------------------------------------------------------ guarded outputs
def _guarded(shape, dtype):
    """A sentinel-filled buffer with MARGIN guard elements on both sides, and the view of `shape` inside it."""
    n = int(np.prod(shape))
    buf = torch.empty(n + 2 * MARGIN, dtype=dtype, device="cuda")
    buf.view(_BITS[dtype]).fill_(_SENT[dtype])
    return buf, buf[MARGIN:MARGIN + n].view(shape)


def _sentinel(t):
    """Elementwise: does t still hold the sentinel bits?"""
    return t.contiguous().view(_BITS[t.dtype]) == _SENT[t.dtype]


def _guarded_call(fn, total_q, H, D, dtype):
    obuf, o = _guarded((total_q, H, D), dtype)
    lbuf, lse = _guarded((H, total_q), torch.float32)
    torch.cuda.synchronize()
    n0 = _capi.launch_count()
    fn(o, lse)
    n = _capi.launch_count() - n0
    torch.cuda.synchronize()
    for buf, what in ((obuf, "O"), (lbuf, "lse")):
        assert bool(_sentinel(buf[:MARGIN]).all()), f"{what}: store before the output"
        assert bool(_sentinel(buf[-MARGIN:]).all()), f"{what}: store past the output"
    return o, lse, n


def _same(a, b):
    return torch.equal(a.nan_to_num(1.0), b.nan_to_num(1.0)) and torch.equal(a.isnan(), b.isnan())


# ------------------------------------------------------------------ one case
def _aim_next(q0, k0, v0, lq, lk, kbn, G):
    """The first kBN keys of sequence b+1 aimed at sequence b's queries: K = 2 sign(sum of b's query rows of the group),
    V = 100 (in place, padded tensors)."""
    for b in range(q0.shape[0] - 1):
        n = min(kbn, lk[b + 1])
        if n == 0 or lq[b] == 0:
            continue
        for hk in range(k0.shape[1]):
            s = q0[b, hk * G:(hk + 1) * G, :lq[b]].float().sum(dim=(0, 1)).sign()
            k0[b + 1, hk, :n] = (2 * s).to(k0.dtype)
            v0[b + 1, hk, :n] = 100.0


class Built:
    """The padded inputs of a case, their packed copies and the two calls."""

    def __init__(self, c, gen, seed, poison):
        self.c, self.gen = c, gen
        dt = _DT[c.dtype]
        B, kbn = len(c.lq), M.kernel_shape(c.D)[0]
        self.B = B
        self.nk = -(-c.max_k // c.page_size) * c.page_size if c.paged else c.max_k
        self.lq, self.lk = V.clamp(c.lq, c.max_q), V.clamp(c.lk, self.nk)
        q0, k0, v0 = _inputs(gen, B, c.H, c.Hkv, c.max_q, self.nk, c.D, None, seed=seed)
        if gen == "randn":
            _aim_next(q0, k0, v0, self.lq, self.lk, kbn, c.H // c.Hkv)
        q16, k16, v16 = _poison(q0, k0, v0, self.lq, self.lk, poison)
        self.q0, self.k0, self.v0 = (x.to(dt) for x in (q0, k0, v0))
        self.qp, self.kp, self.vp = (x.to(dt) for x in (q16, k16, v16))
        self.cu_q = V.offsets(c.lq)
        self.total_q = self.cu_q[-1] + 5
        self.q = V.pack(self.qp, self.cu_q, self.lq, self.total_q, float("nan"))
        self.tq = _lens(self.cu_q)
        if c.paged:
            kpool, vpool, self.table = paginate(k16, v16, self.lk, c.page_size, self.nk // c.page_size, poison,
                                                seed=seed + 1)
            self.k, self.v = kpool.to(dt), vpool.to(dt)
            self.tk = _lens(c.lk)
        else:
            self.cu_k = V.offsets(c.lk)
            total_k = self.cu_k[-1] + 5
            self.k = V.pack(self.kp, self.cu_k, self.lk, total_k, poison)
            self.v = V.pack(self.vp, self.cu_k, self.lk, total_k, poison)
            self.tk = _lens(self.cu_k)
            self.table = None

    def call(self, o, lse):
        c = self.c
        if c.paged:
            flash_attn.fmha_varlen_fwd(self.q, self.k, self.v, o, self.tq, None, c.max_q, 0, causal=c.causal, lse=lse,
                                       block_table=self.table, seqused_k=self.tk)
        else:
            flash_attn.fmha_varlen_fwd(self.q, self.k, self.v, o, self.tq, self.tk, c.max_q, c.max_k, causal=c.causal,
                                       lse=lse)

    def run(self):
        return _guarded_call(self.call, self.total_q, self.c.H, self.c.D, _DT[self.c.dtype])

    def padded(self):
        """The seqlens (paged) call on the padded copies, num_splits = 1."""
        c = self.c
        o = torch.empty_like(self.qp)
        lse = torch.empty(self.qp.shape[:3], device="cuda")
        tq = _lens(self.lq)
        if c.paged:
            flash_attn.fmha_fwd(self.qp, self.k, self.v, o, lse=lse, causal=c.causal, num_splits=1, seqlens_q=tq,
                                seqlens_k=self.tk, block_table=self.table)
        else:
            flash_attn.fmha_fwd(self.qp, self.kp, self.vp, o, lse=lse, causal=c.causal, num_splits=1, seqlens_q=tq,
                                seqlens_k=_lens(self.lk))
        return o, lse


def _check_case(bt, o, lse, key, what):
    c = bt.c
    rows, po, pl = V.unpad_rows(*bt.padded(), bt.cu_q, bt.lq)
    rows = rows.cuda()
    assert torch.equal(o[rows], po) and torch.equal(lse[:, rows], pl), what + ": not bitwise the padded call"
    free = torch.ones(bt.total_q, dtype=torch.bool, device="cuda")
    free[rows] = False
    assert bool(_sentinel(o[free]).all()), what + ": a row of o that no sequence owns was written"
    assert bool(_sentinel(lse[:, free]).all()), what + ": a column of lse that no sequence owns was written"
    # back to the padded layout, padded rows empty (O = 0, lse = -inf), against the fp64 reference
    go = torch.zeros(bt.B, c.H, c.max_q, c.D, device="cuda", dtype=o.dtype)
    gl = torch.full((bt.B, c.H, c.max_q), -math.inf, device="cuda")
    for b in range(bt.B):
        n = bt.lq[b]
        go[b, :, :n] = o[bt.cu_q[b]:bt.cu_q[b] + n].transpose(0, 1)
        gl[b, :, :n] = lse[:, bt.cu_q[b]:bt.cu_q[b] + n]
    sc, poly = R.kernel_scale(c.D), c.D <= 128
    ref = S.reference(bt.q0, bt.k0, bt.v0, sc, c.causal, bt.lq, bt.lk, M.exact_scores(bt.gen))
    bounds = BF if c.dtype == "bf16" else R
    ob, lb = bounds.o_bound(ref, poly)[1], bounds.lse_bound(ref, poly)
    empty = ref["empty"]
    for name, g, w, bd in (("O", go, ref["o"], ob), ("lse", gl, ref["lse"], lb)):
        assert not bool(torch.isnan(g).any()), f"{what} {name}: NaN"
        if bool(empty.any()):
            assert bool((g[empty] == (-math.inf if name == "lse" else 0)).all()), f"{what} {name}: empty row"
        ne = ~empty
        err = (g.double()[ne] - w[ne]).abs()
        if err.numel() == 0:
            continue
        ratio = torch.nan_to_num(err / bd[ne], nan=float("inf")).max().item()
        _ratios[(key, name)] = max(_ratios[(key, name)], ratio)
        assert bool((err <= bd[ne]).all()), f"{what} {name}: |err|/bound {ratio:.3g}"


@pytest.mark.parametrize("i", range(len(V.CASES_BY_SHAPE)),
                         ids=lambda i: "case{}-D{}-{}{}{}".format(i, V.CASES_BY_SHAPE[i].D, V.CASES_BY_SHAPE[i].dtype,
                                                                  "-causal" if V.CASES_BY_SHAPE[i].causal else "",
                                                                  "-paged" if V.CASES_BY_SHAPE[i].paged else ""))
def test_case(i):
    c = V.CASES_BY_SHAPE[i]
    key = V.case_key(c)
    for j, gen in enumerate(c.gens):
        poison = _POISON[(i + j) % len(_POISON)]
        what = (f"{label(key)}: H{c.H} Hkv{c.Hkv} D{c.D} max_q{c.max_q} max_k{c.max_k} page{c.page_size} {gen} "
                f"pad={poison}")
        bt = Built(c, gen, seed=7919 * i + j, poison=poison)
        ins = [x.clone() for x in (bt.q, bt.k, bt.v, bt.tq, bt.tk)] + ([bt.table.clone()] if c.paged else [])
        o, lse, n = bt.run()
        assert n == 1, f"{what}: {n} launches"
        after = [bt.q, bt.k, bt.v, bt.tq, bt.tk] + ([bt.table] if c.paged else [])
        assert all(_same(a, b) for a, b in zip(ins, after)), what + ": an input changed"
        _check_case(bt, o, lse, key, what)


# ------------------------------------------------------------------ kernel names
def _profile_all_cases():
    """Child process: the CUDA kernel names of every case, as one JSON line on stdout."""
    import json
    fns = []
    for i, c in enumerate(V.CASES_BY_SHAPE):
        bt = Built(c, "randn", seed=i, poison=0.0)
        o = torch.empty(bt.total_q, c.H, c.D, device="cuda", dtype=_DT[c.dtype])
        lse = torch.empty(c.H, bt.total_q, device="cuda")
        fns.append(lambda bt=bt, o=o, lse=lse: bt.call(o, lse))
    print("KERNEL_NAMES " + json.dumps(_kernels_per_call(fns)))


@pytest.fixture(scope="module")
def profiled_names():
    return profiled_names_of("test_attn_varlen_gpu")


@pytest.mark.parametrize("i", range(len(V.CASES_BY_SHAPE)))
def test_kernel_names(profiled_names, i):
    c = V.CASES_BY_SHAPE[i]
    key = V.case_key(c)
    names = profiled_names[i] if i < len(profiled_names) else []
    assert names, f"{label(key)}: the profiler recorded no kernel"
    assert len(names) == 1 and V.parse_instantiations(names) == [key], f"{label(key)}: ran {names}"
    assert not any("memcpy" in n.lower() or "dtoh" in n.lower() for n in names), names


# ------------------------------------------------------------------ graphs and streams
@pytest.mark.parametrize("paged", [False, True], ids=["packed", "paged"])
@pytest.mark.parametrize("dtype", ["fp16", "bf16"])
def test_graph_replay_with_new_offsets_and_side_stream(paged, dtype):
    """A captured call replays with new offsets, lengths and tables written into the same tensors, bit for bit the
    eager call; a call on a side stream equals the eager one."""
    c = V.Case(16, 4, 128, True, paged, dtype, (300, 5, 0, 129, 64, 1), (700, 40, 3, 129, 0, 65), 512, 1024,
               16 if paged else None, ("randn",))
    bt = Built(c, "randn", seed=11, poison=float("nan"))
    o = torch.empty(bt.total_q, c.H, c.D, device="cuda", dtype=_DT[dtype])
    lse = torch.empty(c.H, bt.total_q, device="cuda")
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            bt.call(o, lse)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    eo, el, _ = bt.run()
    rows = torch.cat([torch.arange(a, a + n) for a, n in zip(bt.cu_q, bt.lq)]).cuda()
    assert torch.equal(o[rows], eo[rows]) and torch.equal(lse[:, rows], el[:, rows]), "side stream differs from eager"
    o.zero_()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        bt.call(o, lse)
    for new_q, new_k, shift in (((80, 80, 80, 80, 80, 98), (500, 2, 300, 1, 64, 0), 1),
                                ((0, 400, 0, 64, 1, 20), (0, 1000, 5, 64, 129, 700), 3)):
        assert sum(new_q) <= bt.total_q
        bt.tq.copy_(_lens(V.offsets(new_q)))
        if paged:
            bt.tk.copy_(_lens(new_k))
            bt.table.copy_(bt.table.roll(shift, 0))
        else:
            bt.tk.copy_(_lens(V.offsets([min(x, 1 + bt.k.shape[0] // 6) for x in new_k])))
        o.zero_()
        graph.replay()
        torch.cuda.synchronize()
        eo, el, _ = bt.run()
        rows = torch.cat([torch.arange(a, a + min(n, c.max_q)) for a, n in zip(V.offsets(new_q), new_q)]).cuda()
        # a rolled table may hand a sequence poisoned (NaN) pages inside its new length: compare NaN-aware
        assert rows.numel() > 0 and _same(o[rows], eo[rows]) and _same(lse[:, rows], el[:, rows]), \
            f"graph replay with offsets {new_q} differs from eager"


# ------------------------------------------------------------------ chunked prefill through merge_attn_states
@pytest.mark.parametrize("dtype", ["fp16", "bf16"])
def test_chunked_prefill_merges_with_merge_attn_states(dtype):
    """New tokens of three sequences against their paged prefix (non-causal) and against themselves (causal, packed),
    merged by merge_attn_states without reshapes, against the fp64 reference of the whole causal sequence.  Bound:
    each part's o_bound and lse_bound through the merge weights, the merge's fp32 arithmetic and its rounding
    (merge_ref.U / FLOOR), as in test_attn_bf16_gpu.test_key_halves_merge_in_bf16."""
    dt = _DT[dtype]
    H, Hkv, D, ps = 8, 2, 128, 64
    prefix, new = [300, 1000, 64], [200, 77, 129]
    B, G = 3, H // Hkv
    g = torch.Generator(device="cuda").manual_seed(5)
    full = [p + n for p, n in zip(prefix, new)]
    qs = [torch.randn(n, H, D, device="cuda", generator=g).to(dt) for n in new]
    ks = [torch.randn(L, Hkv, D, device="cuda", generator=g).to(dt) for L in full]
    vs = [torch.randn(L, Hkv, D, device="cuda", generator=g).to(dt) for L in full]
    q = torch.cat(qs)
    cu_q = _lens(V.offsets(new))
    total = q.shape[0]
    # the prefix in a paged pool
    maxp = -(-max(prefix) // ps)
    kpad = torch.zeros(B, Hkv, maxp * ps, D, device="cuda", dtype=torch.float16)
    vpad = torch.zeros_like(kpad)
    for b in range(B):
        kpad[b, :, :prefix[b]] = ks[b][:prefix[b]].transpose(0, 1).to(torch.float16)
        vpad[b, :, :prefix[b]] = vs[b][:prefix[b]].transpose(0, 1).to(torch.float16)
    kpool, vpool, table = paginate(kpad, vpad, prefix, ps, maxp, float("nan"), seed=6, pad=-1)
    kpool, vpool = kpool.to(dt), vpool.to(dt)
    oa, la = torch.empty_like(q), torch.empty(H, total, device="cuda")
    flash_attn.fmha_varlen_fwd(q, kpool, vpool, oa, cu_q, None, max(new), 0, lse=la, block_table=table,
                               seqused_k=_lens(prefix))
    # the new tokens' own keys, packed
    kn = torch.cat([k[p:] for k, p in zip(ks, prefix)])
    vn = torch.cat([v[p:] for v, p in zip(vs, prefix)])
    ob, lb = torch.empty_like(q), torch.empty(H, total, device="cuda")
    flash_attn.fmha_varlen_fwd(q, kn, vn, ob, cu_q, cu_q, max(new), max(new), causal=True, lse=lb)
    merged, merged_lse = torch.empty_like(q), torch.empty(H, total, device="cuda")
    MA.merge_attn_states_cuda(merged, oa, la, ob, lb, merged_lse)
    torch.cuda.synchronize()
    sc, poly = R.kernel_scale(D), True
    bounds = BF if dtype == "bf16" else R
    for b in range(B):
        rows = slice(V.offsets(new)[b], V.offsets(new)[b + 1])
        qb = qs[b].transpose(0, 1)[None]                                     # [1, H, n, D]
        kb, vb = ks[b].transpose(0, 1)[None], vs[b].transpose(0, 1)[None]    # [1, Hkv, L, D]
        ke, ve = SR.expand(kb, G), SR.expand(vb, G)
        i = torch.arange(new[b], device="cuda")[:, None] + prefix[b]
        j = torch.arange(full[b], device="cuda")[None, :]
        ref = SR.masked_reference(qb, ke, ve, sc, (j <= i)[None, None])
        ra = SR.masked_reference(qb, ke[:, :, :prefix[b]], ve[:, :, :prefix[b]], sc,
                                 torch.ones(new[b], prefix[b], dtype=torch.bool, device="cuda")[None, None])
        rb = SR.masked_reference(qb, ke[:, :, prefix[b]:], ve[:, :, prefix[b]:], sc,
                                 (j[:, :new[b]] <= i - prefix[b])[None, None])
        wa = 1.0 / (1.0 + torch.exp(rb["lse"] - ra["lse"]))[..., None]
        wb = 1.0 - wa
        ba, bb = bounds.o_bound(ra, poly)[1], bounds.o_bound(rb, poly)[1]
        dl = (bounds.lse_bound(ra, poly) + bounds.lse_bound(rb, poly))[..., None]
        bound = (wa * ba + wb * bb + wa * wb * dl * (ra["o"] - rb["o"]).abs()
                 + 2.0 ** -20 * (wa * ra["o"].abs() + wb * rb["o"].abs()) + MR.U[dt] * ref["o"].abs() + MR.FLOOR[dt])
        err = (merged[rows].transpose(0, 1)[None].double() - ref["o"]).abs()
        ratio = (err / bound).max().item()
        _ratios[(("merge", dtype), "O")] = max(_ratios[(("merge", dtype), "O")], ratio)
        assert bool((err <= bound).all()), f"sequence {b}: |err|/bound {ratio:.3g}"
        lse_err = (merged_lse[:, rows][None].double() - ref["lse"]).abs()
        assert bool((lse_err <= bounds.lse_bound(ref, poly) + bounds.lse_bound(ra, poly) + bounds.lse_bound(rb, poly)
                     + 2.0 ** -20).all()), f"sequence {b}: lse"


# ------------------------------------------------------------------ the benchmarked shapes
def _bench_tool():
    path = Path(__file__).resolve().parents[1] / "tools" / "bench_attn_varlen.py"
    spec = importlib.util.spec_from_file_location("bench_attn_varlen", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


_TOOL = _bench_tool()


@pytest.mark.parametrize("index", range(len(_TOOL.SHAPES)), ids=lambda i: _TOOL.SHAPES[i][0].replace(" ", "-"))
def test_benchmarked_shape(index):
    """Every shape of tools/bench_attn_varlen.py at full size, with its seeded lengths: bit for bit the padded call."""
    name, B, H, Hkv, D, causal, _, nq, ps = _TOOL.SHAPES[index]
    lq, lk = _TOOL.lengths(index)
    mq, mk = max(lq), max(lk)
    mk = -(-mk // ps) * ps if ps else mk   # whole pages for paginate
    g = torch.Generator(device="cuda").manual_seed(300 + index)
    qp = torch.randn(B, H, mq, D, device="cuda", generator=g).half()
    kp = torch.randn(B, Hkv, mk, D, device="cuda", generator=g).half()
    vp = torch.randn(B, Hkv, mk, D, device="cuda", generator=g).half()
    cq = V.offsets(lq)
    q = V.pack(qp, cq, lq, cq[-1], 0.0)
    o, lse = torch.empty_like(q), torch.empty(H, cq[-1], device="cuda")
    po, pl = torch.empty_like(qp), torch.empty(B, H, mq, device="cuda")
    n0 = _capi.launch_count()
    if ps is None:
        ck = V.offsets(lk)
        k, v = V.pack(kp, ck, lk, ck[-1], 0.0), V.pack(vp, ck, lk, ck[-1], 0.0)
        flash_attn.fmha_varlen_fwd(q, k, v, o, _lens(cq), _lens(ck), mq, max(lk), causal=causal, lse=lse)
        assert _capi.launch_count() - n0 == 1
        flash_attn.fmha_fwd(qp, kp, vp, po, lse=pl, causal=causal, seqlens_q=_lens(lq), seqlens_k=_lens(lk))
    else:
        kc, vc, table = paginate(kp, vp, lk, ps, -(-mk // ps), float("nan"), seed=index, pad=-1)
        flash_attn.fmha_varlen_fwd(q, kc, vc, o, _lens(cq), None, mq, 0, causal=causal, lse=lse, block_table=table,
                                   seqused_k=_lens(lk))
        assert _capi.launch_count() - n0 == 1
        flash_attn.fmha_fwd(qp, kc, vc, po, lse=pl, causal=causal, seqlens_q=_lens(lq), seqlens_k=_lens(lk),
                            block_table=table)
    rows, wo, wl = V.unpad_rows(po, pl, cq, lq)
    assert torch.equal(o, wo) and torch.equal(lse, wl), f"{name}: not bitwise the padded call"
    assert not bool(o.isnan().any())
