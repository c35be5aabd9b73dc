"""Every workload of bench_workloads.WORKLOADS whose check is here, run the way its benchmark runs it (the same op
names and arguments) at the shape it is timed at, into NaN guard bands (test_attn_numerics_gpu._guarded), and checked:

* fp64 per-element bounds: attention against attn_ref.o_bound / lse_bound (split calls: attn_split_ref.combine_bound
  of the key ranges of the split count the call used, per-sequence lengths: attn_seqlens_ref's ranges), the fused RMS
  norm against attn_ref.rms_reference, the unfused pair's rms_norm against rope_rms_ref.rms_reference of its input,
  GEMM against gemm_ref.  References are computed on the GPU in float64, per sequence.  Rows: decoding (Nq <= 16) all
  of them; otherwise, in every (batch, head), the first and last row of every query tile, both sides of the boundary
  between its two consumer warpgroups, and with the mask the rows where the diagonal enters a new key block, so every
  CTA is checked.  Per-sequence lengths: those rows below Lq_b (row 0 and Lq_b - 1 among them), and every padded row
  exactly O = 0, lse = -inf.  The bench ops take no lse: a second call with lse must give the same O bit for bit.
* a gather probe over the whole tensor: q_i = c code(k_t) (attn_ref's one_hot codes, >= 48 nats above every other
  key) with t random among the visible keys, t = i + diag with the mask (attn_mask_ref's diag_gather): O_i = V_t to
  one fp16 ulp in every row of every head.
* bit for bit: the host-buffer entries against the device calls, GQA num_splits=1 against the expanded K/V call,
  the seqlens call against the call on one sequence alone (shortest, longest and two others), the 16384^3 GEMM against
  its two row shards (b200_hgemm_f16_rows) and the fused all-gather epilogue with local buffers standing in for the
  peer, and the bench's back-to-back launches over its rotating operand sets against isolated calls.

test_split_counts checks b200_fmha_fwd_f16_gqa_splits against bench_workloads.auto_splits and, on 132 SMs, against the
README.  The largest |err| / bound per workload, the peak device memory and the module time are printed at the end
(pytest -s).
"""
import collections
import ctypes
import math
import time
import zlib

import numpy as np
import pytest
import torch

import attn_mask_ref as M
import attn_ref as R
import attn_seqlens_ref as SQ
import attn_split_ref as SR
import bench_workloads as W
import gemm_ref as GR
import rope_rms_ref as RR
from leetcuda_b200 import _capi, ffpa_attn, flash_attn, fused_ops, hgemm, rms_norm
from test_attn_numerics_gpu import _assert_margins, _guarded
from test_gemm_numerics_gpu import _sample_rows

pytestmark = pytest.mark.gpu

_ratios = collections.defaultdict(float)


@pytest.fixture(scope="module", autouse=True)
def _report():
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    yield
    if _ratios:
        print("\nlargest |err| / bound per workload (attn_ref, attn_split_ref, rope_rms_ref, gemm_ref):")
        for wid in sorted({k for k, _ in _ratios}):
            parts = "  ".join(f"{q} {_ratios[(w, q)]:.3f}" for w, q in sorted(_ratios) if w == wid)
            print(f"  {wid:<72} {parts}")
    print(f"peak device memory {torch.cuda.max_memory_allocated() / 2 ** 30:.1f} GiB")
    print(f"module time {time.time() - t0:.1f} s")


def _seed(wid, salt=0):
    return zlib.crc32(wid.encode()) + salt


def _gen(wid, salt=0):
    return torch.Generator(device="cuda").manual_seed(_seed(wid, salt))


def _check(wid, name, got, want, bound, what, empty=None):
    """got within bound of want elementwise; rows marked empty exactly O = 0 / lse = -inf."""
    assert not bool(torch.isnan(got).any()), f"{what} {name}: NaN"
    if empty is not None and bool(empty.any()):
        assert bool((got[empty] == (-math.inf if name == "lse" else 0)).all()), f"{what} {name}: empty row"
        ne = ~empty
        got, want, bound = got[ne], want[ne], bound[ne]
    if got.numel() == 0:
        return
    err = (got.double() - want).abs()
    r = torch.nan_to_num(err / bound, nan=math.inf)
    ratio = r.max().item()
    _ratios[(wid, name)] = max(_ratios[(wid, name)], ratio)
    if not bool((err <= bound).all()):
        i = int(r.reshape(-1).argmax())
        pytest.fail(f"{what} {name}: |err|/bound {ratio:.3g}: got {got.reshape(-1)[i].item()}, "
                    f"want {want.reshape(-1)[i].item()}")


# ------------------------------------------------------------------ attention: the calls
_BENCH_OPS = {"flash_attn_mma_stages_split_q_shared_qkv": flash_attn, "ffpa_mma_acc_f32_L1": ffpa_attn}


def _splits(c, B, Nq, Nk):
    s = c["num_splits"]
    return s or _capi.lib().b200_fmha_fwd_f16_gqa_splits(B, c["H"], c["Hkv"], Nq, Nk, c["D"])


def _lens_t(c):
    lens = c["lens"]
    if lens is None:
        return None, None
    return tuple(torch.tensor(x, dtype=torch.int32, device="cuda") for x in lens)


def _run(c, q, k, v, what):
    """The workload's call on q, k, v ([B,Hkv,..] K/V; expanded here when the workload expands) into a guarded O, then
    the same call with lse into guarded O and lse: O must agree bit for bit.  Returns (O, lse)."""
    G = c["H"] // c["Hkv"]
    if c["expanded"]:
        k, v = k.repeat_interleave(G, 1).contiguous(), v.repeat_interleave(G, 1).contiguous()
    tq, tk = _lens_t(c)
    obuf, o = _guarded(tuple(q.shape), torch.float16)
    if c["op"] in _BENCH_OPS:
        getattr(_BENCH_OPS[c["op"]], c["op"])(q, k, v, o, 2)
    else:
        assert c["op"] == "fmha_fwd", c["op"]
        kw = {} if c["lens"] is None else {"seqlens_q": tq, "seqlens_k": tk}
        flash_attn.fmha_fwd(q, k, v, o, causal=c["causal"], num_splits=c["num_splits"], **kw)
    o2buf, o2 = _guarded(tuple(q.shape), torch.float16)
    lbuf, lse = _guarded(tuple(q.shape[:3]), torch.float32)
    flash_attn.fmha_fwd(q, k, v, o2, lse=lse, causal=c["causal"], num_splits=c["num_splits"], seqlens_q=tq,
                        seqlens_k=tk)
    torch.cuda.synchronize()
    for buf, name in ((obuf, "O"), (o2buf, "O with lse"), (lbuf, "lse")):
        _assert_margins(buf, f"{what} {name}")
    assert torch.equal(o, o2), f"{what}: O differs between the call without and with lse"
    return o, lse


def _run_loop(c, q, k, v, what):
    """The seqlens tool's loop: one fmha_fwd(..., num_splits=0) per sequence on its sliced tensors, each into its own
    guarded output.  Returns [(O_b, lse_b)] (lse from a second call per sequence, O checked equal)."""
    lq, lk = c["lens"]
    out = []
    for b in range(q.shape[0]):
        qs = q[b:b + 1, :, :lq[b]].contiguous()
        ks, vs = k[b:b + 1, :, :lk[b]].contiguous(), v[b:b + 1, :, :lk[b]].contiguous()
        sub = dict(c, op="fmha_fwd", B=1, Nq=lq[b], Nk=lk[b], lens=None)
        out.append(_run(sub, qs, ks, vs, f"{what} sequence {b}"))
    return out


# ------------------------------------------------------------------ attention: fp64 bounds
def _rows(lq, diag, D, causal):
    """Query rows to check below lq (see the module docstring)."""
    if lq <= 16:
        return list(range(lq))
    kbn, per = M.kernel_shape(D)
    rows = set()
    for t0 in range(0, lq, per):
        rows |= {t0, min(t0 + per, lq) - 1}
        if per == 128:
            rows |= {t0 + 63, t0 + 64}
    if causal:
        for i in range(lq):
            if (i + diag) % kbn == 0:
                rows |= {i - 1, i}
    return sorted(r for r in rows if 0 <= r < lq)


def _check_sequence(wid, c, o, lse, q, k, v, lq, lk, splits, what):
    """One sequence: o, lse [1,H,Nq,..] from q [1,H,Nq,D], k, v [1,Hkv,Nk,D] with lq queries and lk keys visible."""
    D, causal, poly, sc = c["D"], c["causal"], c["D"] <= 128, R.kernel_scale(c["D"])
    G = q.shape[1] // k.shape[1]
    if splits > 1:
        assert q.shape[2] <= 16, f"{what}: a split call is checked on all rows"
        parts = SQ.part_references(q, k, v, sc, causal, splits, [lq], [lk])
        want_o, want_l, empty, ob, lb = SR.combine_bound(parts, poly)
        _check(wid, "O", o, want_o, ob, what, empty)
        _check(wid, "lse", lse, want_l, lb, what, empty)
        return
    rows = _rows(lq, lk - lq, D, causal)
    r = torch.tensor(rows, device="cuda")
    i, j = r[:, None], torch.arange(k.shape[2], device="cuda")[None, :]
    vis = (i < lq) & (j < lk)
    if causal:
        vis &= j <= i + (lk - lq)
    ref = SR.masked_reference(q[:, :, r], SR.expand(k, G), SR.expand(v, G), sc, vis[None, None])
    _, ob = R.o_bound(ref, poly)
    _check(wid, "O", o[:, :, r], ref["o"], ob, what, ref["empty"])
    _check(wid, "lse", lse[:, :, r], ref["lse"], R.lse_bound(ref, poly), what, ref["empty"])


def _lengths(c):
    B = c["B"]
    return c["lens"] if c["lens"] is not None else ((c["Nq"],) * B, (c["Nk"],) * B)


def _check_padded_rows(c, o, lse, what):
    lq, _ = c["lens"]
    for b in range(c["B"]):
        assert bool((o[b, :, lq[b]:] == 0).all()), f"{what}: padded rows of sequence {b} are not 0"
        assert bool((lse[b, :, lq[b]:] == -math.inf).all()), f"{what}: padded rows of sequence {b}: lse not -inf"


def _attention_fp64(wid, c):
    B, H, Hkv, Nq, Nk, D = (c[x] for x in ("B", "H", "Hkv", "Nq", "Nk", "D"))
    g = _gen(wid)
    q = torch.randn(B, H, Nq, D, device="cuda", dtype=torch.half, generator=g)
    k, v = (torch.randn(B, Hkv, Nk, D, device="cuda", dtype=torch.half, generator=g) for _ in range(2))
    lq, lk = _lengths(c)
    what = f"{wid} randn"
    if c["op"] == "fmha_fwd_loop":
        for b, (o, lse) in enumerate(_run_loop(c, q, k, v, what)):
            qs, ks, vs = q[b:b + 1, :, :lq[b]], k[b:b + 1, :, :lk[b]], v[b:b + 1, :, :lk[b]]
            _check_sequence(wid, c, o, lse, qs, ks, vs, lq[b], lk[b], _splits(c, 1, lq[b], lk[b]),
                            f"{what} sequence {b}")
        return
    o, lse = _run(c, q, k, v, what)
    S = _splits(c, B, Nq, Nk)
    for b in range(B):
        _check_sequence(wid, c, o[b:b + 1], lse[b:b + 1], q[b:b + 1], k[b:b + 1], v[b:b + 1], lq[b], lk[b], S,
                        f"{what} sequence {b}")
    if c["lens"] is not None:
        _check_padded_rows(c, o, lse, what)
        _unsplit_sequences_are_bitwise(c, q, k, v, what)
    if c["expanded"]:
        o2, l2 = _run(dict(c, expanded=False, num_splits=1), q, k, v, what + " num_splits=1")
        assert torch.equal(o, o2) and torch.equal(lse, l2), f"{what}: num_splits=1 and expanded K/V differ"


def _unsplit_sequences_are_bitwise(c, q, k, v, what):
    """The seqlens call without a split against fmha_fwd on one sequence alone: the shortest, the longest and two
    others (by key length), bit for bit."""
    lq, lk = c["lens"]
    o, lse = _run(dict(c, num_splits=1), q, k, v, what + " num_splits=1")
    order = sorted(range(c["B"]), key=lambda b: lk[b])
    pick = sorted({order[0], order[-1], order[len(order) // 3], order[2 * len(order) // 3]})
    for b in pick:
        qs = q[b:b + 1, :, :lq[b]].contiguous()
        ks, vs = k[b:b + 1, :, :lk[b]].contiguous(), v[b:b + 1, :, :lk[b]].contiguous()
        one = dict(c, op="fmha_fwd", B=1, Nq=lq[b], Nk=lk[b], lens=None, num_splits=1)
        os_, ls = _run(one, qs, ks, vs, f"{what} sequence {b} alone")
        assert torch.equal(o[b:b + 1, :, :lq[b]], os_) and torch.equal(lse[b:b + 1, :, :lq[b]], ls), \
            f"{what}: sequence {b} (Lq {lq[b]}, Lk {lk[b]}) is not bitwise the call on it alone"


# ------------------------------------------------------------------ attention: the gather probe
def _gather_inputs(wid, c):
    """Keys are distinct +-1 codes (attn_ref's one_hot: the first bits spell the key index), q_i = c code(k_t) with t
    a random visible key, or t = i + diag with the mask.  Returns q, k, v, the targets [B,H,Nq] and the rows that see a
    key."""
    B, H, Hkv, Nq, Nk, D = (c[x] for x in ("B", "H", "Hkv", "Nq", "Nk", "D"))
    G = H // Hkv
    g = _gen(wid, 1)
    codes = (torch.randint(0, 2, (B, Hkv, Nk, D), device="cuda", generator=g, dtype=torch.int8) * 2 - 1).half()
    nb = max(1, (Nk - 1).bit_length())
    assert nb <= D
    j = torch.arange(Nk, device="cuda")[:, None]
    codes[..., :nb] = (((j >> torch.arange(nb, device="cuda")) & 1) * 2 - 1).half()
    v = torch.randn(B, Hkv, Nk, D, device="cuda", dtype=torch.half, generator=g)
    lq, lk = _lengths(c)
    lqt = torch.tensor(lq, device="cuda")[:, None, None]
    lkt = torch.tensor(lk, device="cuda")[:, None, None]
    i = torch.arange(Nq, device="cuda")[None, None, :]
    if c["causal"]:
        t = (i + lkt - lqt).expand(B, H, Nq)
    else:
        t = (torch.rand(B, H, Nq, device="cuda", generator=g) * lkt).long().clamp(max=Nk - 1)
    valid = (i < lqt) & (t >= 0)
    t = torch.where(valid, t, 0)
    bi = torch.arange(B, device="cuda")[:, None, None]
    hk = (torch.arange(H, device="cuda") // G)[None, :, None]
    scale = float(np.float16(24.0 / R.kernel_scale(D)))
    q = (codes[bi, hk, t].float() * scale).half()
    q[~valid.expand(B, H, Nq)] = 0
    return q, codes, v, v[bi, hk, t].double(), valid.expand(B, H, Nq)


def _assert_gathered(o, truth, valid, what):
    ulp = torch.exp2(torch.floor(torch.log2(truth.abs().clamp_min(2.0 ** -14))) - 10)
    ok = ((o.double() - truth).abs() <= ulp).all(-1)
    bad = valid & ~ok
    assert not bool(bad.any()), f"{what}: O is not the gathered V in {int(bad.sum())} rows, first {bad.nonzero()[0].tolist()}"
    assert bool((o[~valid] == 0).all()), f"{what}: rows without a visible key are not 0"


def _attention_gather(wid, c):
    q, k, v, truth, valid = _gather_inputs(wid, c)
    what = f"{wid} gather"
    if c["op"] == "fmha_fwd_loop":
        lq, _ = c["lens"]
        for b, (o, _) in enumerate(_run_loop(c, q, k, v, what)):
            _assert_gathered(o, truth[b:b + 1, :, :lq[b]], valid[b:b + 1, :, :lq[b]], f"{what} sequence {b}")
        return
    o, _ = _run(c, q, k, v, what)
    _assert_gathered(o, truth, valid, what)


def _bench_rotation(wid, c):
    """bench.attention_row: nsets operand sets and outputs, launched back to back (i % nsets); every output bit-equal
    to an isolated call on its set."""
    B, H, N, D = c["B"], c["H"], c["Nq"], c["D"]
    op = getattr(_BENCH_OPS[c["op"]], c["op"])
    n = c["sets"]
    g = _gen(wid, 2)
    sets = [[torch.randn(B, H, N, D, device="cuda", dtype=torch.half, generator=g) for _ in range(3)] for _ in range(n)]
    outs = [torch.empty(B, H, N, D, device="cuda", dtype=torch.half) for _ in range(n)]
    for i in range(3 * n + 1):
        op(*sets[i % n], outs[i % n], 2)
    torch.cuda.synchronize()
    for j in range(n):
        iso = torch.empty_like(outs[j])
        op(*sets[j], iso, 2)
        torch.cuda.synchronize()
        assert torch.equal(outs[j], iso), f"{wid}: set {j} after back-to-back launches differs from an isolated call"


def _attention(wid, c):
    _attention_fp64(wid, c)
    _attention_gather(wid, c)
    if c["sets"]:
        _bench_rotation(wid, c)


# ------------------------------------------------------------------ host-buffer attention
def _fmha_host(wid, c):
    B, H, N, D = c["B"], c["H"], c["N"], c["D"]
    g = torch.Generator().manual_seed(_seed(wid))
    hq, hk, hv = (torch.randn(B, H, N, D, generator=g).half().pin_memory() for _ in range(3))
    ho = torch.full((B, H, N, D), float("nan"), dtype=torch.half).pin_memory()
    flash_attn.fmha_host(hq, hk, hv, ho)
    q, k, v = (x.cuda() for x in (hq, hk, hv))
    obuf, o = _guarded((B, H, N, D), torch.float16)
    getattr(_BENCH_OPS[c["device_op"]], c["device_op"])(q, k, v, o, 2)
    torch.cuda.synchronize()
    _assert_margins(obuf, wid)
    assert torch.equal(ho, o.cpu()), f"{wid}: the host-buffer entry differs from the device call"


# ------------------------------------------------------------------ the RMS-norm epilogue and its unfused pair
def _rms(wid, c):
    B, H, N, D, gain = c["B"], c["H"], c["N"], c["D"], c["g"]
    g = _gen(wid)
    sets = [[torch.randn(B, H, N, D, device="cuda", dtype=torch.half, generator=g) for _ in range(3)] for _ in range(2)]
    obuf, o = _guarded((B, H, N, D), torch.float16)
    o2buf, o2 = _guarded((B, H, N, D), torch.float16)
    fused = c["op"] == "attn_rmsnorm"

    def step(i, o, o2):
        if fused:
            fused_ops.attn_rmsnorm(*sets[i % 2], o, gain)
        else:
            flash_attn.fmha_fwd(*sets[i % 2], o)
            rms_norm.rms_norm(o.view(-1, D), o2.view(-1, D), gain)

    steps = 5                                   # back to back over the two sets, as bench_rows times them
    for i in range(steps):
        step(i, o, o2)
    torch.cuda.synchronize()
    _assert_margins(obuf, wid + " O")
    _assert_margins(o2buf, wid + " rms_norm out")
    last = (steps - 1) % 2
    iso, iso2 = torch.empty_like(o), torch.empty_like(o2)
    step(last, iso, iso2)
    torch.cuda.synchronize()
    assert torch.equal(o, iso) and (fused or torch.equal(o2, iso2)), f"{wid}: back-to-back differs from isolated"
    q, k, v = sets[last]
    lbuf, lse = _guarded((B, H, N), torch.float32)
    o3 = torch.empty_like(o)
    if fused:
        fused_ops.attn_rmsnorm(q, k, v, o3, gain, lse=lse)
    else:
        flash_attn.fmha_fwd(q, k, v, o3, lse=lse)
    torch.cuda.synchronize()
    _assert_margins(lbuf, wid + " lse")
    assert torch.equal(o3, o), f"{wid}: O differs between the call without and with lse"
    sc, rows = R.kernel_scale(D), torch.tensor(_rows(N, 0, D, False), device="cuda")
    for b in range(B):
        ref = R.reference(q[b:b + 1, :, rows], k[b:b + 1], v[b:b + 1], sc)
        pre, ob = R.o_bound(ref, poly=D <= 128)
        want, bound = (R.rms_reference(ref, gain, pre) if fused else (ref["o"], ob))
        _check(wid, "O", o[b:b + 1, :, rows], want, bound, f"{wid} sequence {b}")
        _check(wid, "lse", lse[b:b + 1, :, rows], ref["lse"], R.lse_bound(ref, poly=D <= 128), f"{wid} sequence {b}")
    if not fused:
        want, bound = RR.rms_reference(o.view(-1, D), gain)
        _check(wid, "rms_norm", o2.view(-1, D), want, bound, wid + " rms_norm of O")


# ------------------------------------------------------------------ GEMM
def _hgemm(wid, c):
    M, N, K, n = c["M"], c["N"], c["K"], c["sets"]
    op = getattr(hgemm, c["op"])
    g = _gen(wid)
    As = [torch.randn(M, K, device="cuda", dtype=torch.half, generator=g) for _ in range(n)]
    Bs = [torch.randn(K, N, device="cuda", dtype=torch.half, generator=g) for _ in range(n)]
    bufs = [_guarded((M, N), torch.float16) for _ in range(1 if c["single_out"] else n)]
    steps = 2 * n + 1
    for i in range(steps):
        op(As[i % n], Bs[i % n], bufs[0 if c["single_out"] else i % n][1], 2, True, 2048)
    torch.cuda.synchronize()
    for buf, _ in bufs:
        _assert_margins(buf, wid)
    check_sets = [(steps - 1) % n] if c["single_out"] else range(n)
    iso = torch.empty(M, N, device="cuda", dtype=torch.half)
    for j in check_sets:
        op(As[j], Bs[j], iso, 2, True, 2048)
        torch.cuda.synchronize()
        got = bufs[0 if c["single_out"] else j][1]
        assert torch.equal(got, iso), f"{wid}: set {j} after back-to-back launches differs from an isolated call"
    a, b, full = As[check_sets[-1]], Bs[check_sets[-1]], iso
    if c["fp64"]:
        rows = _sample_rows(M)
        ref = GR.reference(a[rows], b, "f16")
        _check(wid, "C", full[rows], ref["c"], GR.bound(ref), wid)
    world = c["shards"]
    if world:
        rows = M // world
        stream = torch.cuda.current_stream().cuda_stream
        cbuf, cfull = _guarded((M, N), torch.float16)
        for r in range(world):
            rc = _capi.lib().b200_hgemm_f16_rows(a[r * rows:(r + 1) * rows].data_ptr(), b.data_ptr(), cfull.data_ptr(),
                                                 rows, N, K, _capi.B_ROW_MAJOR_KN, r * rows, stream)
            assert rc == 0, _capi.last_error()
        torch.cuda.synchronize()
        _assert_margins(cbuf, wid + " rows")
        assert torch.equal(cfull, full), f"{wid}: the {world} row shards differ from the single-GPU product"
        del cbuf, cfull
        # the fused all-gather epilogue: rank r's C and the peers' C are local buffers here
        own = [_guarded((M, N), torch.float16) for _ in range(world)]
        for r in range(world):
            peers = [own[p][1] for p in range(world) if p != r]
            arr = (ctypes.c_void_p * len(peers))(*[p.data_ptr() for p in peers])
            rc = _capi.lib().b200_hgemm_f16_rows_fused(a[r * rows:(r + 1) * rows].data_ptr(), b.data_ptr(),
                                                       own[r][1].data_ptr(), None, arr, len(peers), rows, N, K,
                                                       _capi.B_ROW_MAJOR_KN, r * rows, stream)
            assert rc == 0, _capi.last_error()
        torch.cuda.synchronize()
        for r, (buf, view) in enumerate(own):
            _assert_margins(buf, f"{wid} fused rank {r}")
            assert torch.equal(view, full), f"{wid}: rank {r}'s C after the fused all-gather differs"


def _hgemm_host(wid, c):
    M, N, K = c["M"], c["N"], c["K"]
    g = torch.Generator().manual_seed(_seed(wid))
    ha = torch.randn(M, K, generator=g).half().pin_memory()
    hb = torch.randn(K, N, generator=g).half().pin_memory()
    hc = torch.full((M, N), float("nan"), dtype=torch.half).pin_memory()
    hgemm.hgemm_host(ha, hb, hc)
    buf, dc = _guarded((M, N), torch.float16)
    getattr(hgemm, c["device_op"])(ha.cuda(), hb.cuda(), dc, 2, True, 2048)
    torch.cuda.synchronize()
    _assert_margins(buf, wid)
    assert torch.equal(hc, dc.cpu()), f"{wid}: the host-buffer entry differs from the device GEMM"


_HANDLERS = {"attention": _attention, "fmha_host": _fmha_host, "rms": _rms, "hgemm": _hgemm,
             "hgemm_host": _hgemm_host}
_HERE = [w for w in W.WORKLOADS if W.GPU_CASE in w.check]


@pytest.mark.parametrize("wid", [w.id for w in _HERE])
def test_workload(wid):
    w = W.BY_ID[wid]
    _HANDLERS[w.call["kind"]](wid, w.call)
    torch.cuda.empty_cache()


def test_split_counts():
    """b200_fmha_fwd_f16_gqa_splits for every num_splits=0 call the tools make (the loop's per sequence) against the
    restated rule, and on 132 SMs the counts the README reports."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    lib = _capi.lib()
    for w in W.WORKLOADS:
        c = w.call
        if c["kind"] != "attention" or c["num_splits"] != 0:
            continue
        calls = ([(1, lq, lk) for lq, lk in zip(*c["lens"])] if c["op"] == "fmha_fwd_loop"
                 else [(c["B"], c["Nq"], c["Nk"])])
        for B, Nq, Nk in calls:
            got = lib.b200_fmha_fwd_f16_gqa_splits(B, c["H"], c["Hkv"], Nq, Nk, c["D"])
            want = W.auto_splits(B, c["H"], c["Hkv"], Nq, Nk, c["D"], sms)
            assert got == want, f"{w.id} B{B} Nq{Nq} Nk{Nk}: the library splits {got} ways, the rule says {want}"
    decode = [lib.b200_fmha_fwd_f16_gqa_splits(B, H, Hkv, Nq, Nk, D) for _, B, H, Hkv, Nq, Nk, D, _ in W.DECODE.SHAPES]
    _, B, H, Hkv, Nq, Nk, D, *_ = W.SEQLENS.SHAPES[1]
    long_decode = lib.b200_fmha_fwd_f16_gqa_splits(B, H, Hkv, Nq, Nk, D)
    print(f"\n{sms} SMs; split counts of the decode tool's SHAPES: {decode}; seqlens B{B} long decode: {long_decode}")
    if sms == 132:
        assert decode == [16, 2, 1, 1, 2, 1, 1] and long_decode == 4, (decode, long_decode)
