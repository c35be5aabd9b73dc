"""A paged serving schedule end to end on the GPU (serve_ref): chunked prefill and graph-captured decode over a reused page
pool, against the fp64 history of every request.

Two copies of the pool run the same schedule.  Pool A is driven by the system under test: every prefill chunk is
fmha_fwd_kvcache(B=1, causal=True) on the request's table row, and every decode step is one fmha_fwd_kvcache(n_new=1)
over all B_MAX slots, captured once in a CUDA graph and replayed with the table, lengths, q, k and v rewritten in place.
Pool B is driven eagerly by the hand-written sequence, kvcache_append(q=, q_out=, seqlens_out=) then fmha_fwd, which also
gives the rotated q of the references.  An e4m3 scenario keeps a third, fp16 / bf16 pool C that receives the same
appends, so every e4m3 row can be checked against the quantisation of the T row.  A page whose last owner finishes is
filled with NaN bits in every pool.  After every call:
  1. A and B agree bit for bit: O, lse, the returned lengths and both pools;
  2. the rows written are the request's tokens at their absolute positions (kvcache_ref's rotary bound, e4m3 bit for bit
     the quantisation of pool C's row, everything else bit for bit), q within the rotary bound, and no other byte of
     the pool changed: other requests' pages, shared prefix pages, freed pages, rows past capacity, idle slots;
  3. every live request's pages, gathered through its table, equal its shadow history bit for bit;
  4. O and lse within the library's per-element bounds of the fp64 attention of the rotated q over the shadow history
     (attn_split_ref.combine_bound when the call splits); an idle slot's O is exactly 0 (its one key reads zeros);
  5. T caches: every prefill chunk through fmha_varlen_fwd(block_table=, seqused_k=) on pool B equals the unsplit paged
     call bit for bit;
  6. at a few decode steps of the request on a shared prefix: attention over the prefix pages and over the rest through
     a shifted table, merged by merge_attn_states, within merge_ref's bound of the fp64 merge of the two parts, and
     each part within its own bound of the fp64 attention over its keys.
The module prints the largest |err| / bound of every scenario and its wall time.
"""
import time

import pytest
import torch

import kvcache_ref as K
import merge_ref as MR
import serve_ref as SV
from leetcuda_b200 import _capi, flash_attn
from leetcuda_b200.merge_attn_states import merge_attn_states_cuda

pytestmark = pytest.mark.gpu

B = SV.B_MAX
MERGE_STEPS = 3
_ratios = {}


@pytest.fixture(scope="module", autouse=True)
def _report():
    t0 = time.time()
    yield
    print("\nlargest |err| / bound per scenario (serve_ref: attention bounds, merge_ref):")
    for nm, r in _ratios.items():
        print(f"  {nm}: " + ", ".join(f"{k} {v:.3g}" for k, v in sorted(r.items())))
    print(f"test_serve_gpu wall time {time.time() - t0:.1f} s")


def _bits32(x):
    return x.view(torch.int32)


def _same(a, b):
    return torch.equal(SV.raw(a), SV.raw(b)) if a.dtype != torch.float32 else torch.equal(_bits32(a), _bits32(b))


def _poison(pools, pages, dt):
    idx = torch.tensor(pages, device="cuda")
    for p in pools:
        SV.raw(p)[idx] = SV.POISON[dt]


def _ok(err):
    assert err is None, err


@pytest.mark.parametrize("i", range(len(SV.SCENARIOS)))
def test_serve(i):
    sc = SV.SCENARIOS[i]
    ratios = _ratios.setdefault(SV.name(sc), {})
    reqs = SV.requests(sc)
    events = SV.schedule(sc, reqs)
    tokens = SV.Tokens(sc, reqs)
    T, dt, e4m3 = K.TORCH[sc.T], SV.dtype(sc), sc.cache == "e4m3"
    H, Hkv, D, ps, mp, cap = sc.H, sc.Hkv, sc.D, sc.page_size, sc.max_pages, SV.capacity(sc)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    gen = torch.Generator().manual_seed(77 + i)
    shape = (SV.num_pages(sc), ps, Hkv, D)
    rd = torch.uint8 if e4m3 else torch.int16
    lo, hi = (0, 256) if e4m3 else (-32768, 32768)
    kA = torch.randint(lo, hi, shape, generator=gen, dtype=torch.int32).to(rd).cuda().view(dt)   # random bits
    vA = torch.randint(lo, hi, shape, generator=gen, dtype=torch.int32).to(rd).cuda().view(dt)
    kB, vB = kA.clone(), vA.clone()
    kC, vC = (torch.zeros(shape, dtype=T, device="cuda") for _ in range(2)) if e4m3 else (None, None)
    prev_k, prev_v = kA.clone(), vA.clone()
    cos, sin = SV.rotary_tables(sc)
    rot = dict(rotary_cos=None if cos is None else cos.cuda(), rotary_sin=None if sin is None else sin.cuda(),
               rotary_interleaved=SV.interleaved(sc))
    scales = dict(k_scale=sc.k_scale, v_scale=sc.v_scale)
    tab = torch.full((B, mp), -1, dtype=torch.int32, device="cuda")
    lens = torch.zeros(B, dtype=torch.int32, device="cuda")
    qd = torch.zeros(B, H, 1, D, dtype=T, device="cuda")
    kd, vd = (torch.zeros(B, Hkv, 1, D, dtype=T, device="cuda") for _ in range(2))
    od = torch.empty_like(qd)
    lsed = torch.empty(B, H, 1, device="cuda")
    dsplit = SV.splits(sc, B, 1, sms)
    assert dsplit == (sc.num_splits or _capi.lib().b200_fmha_fwd_f16_gqa_splits(B, H, Hkv, 1, cap, D))
    step_kw = dict(block_table=tab, lse=lsed, num_splits=sc.num_splits, **rot, **scales)
    # every slot idle (table -1, lengths 0): the warm-up stores nothing
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        flash_attn.fmha_fwd_kvcache(qd, kA, vA, od, kd, vd, lens, **step_kw)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        lens_out = flash_attn.fmha_fwd_kvcache(qd, kA, vA, od, kd, vd, lens, **step_kw)
    torch.cuda.synchronize()
    assert _same(kA, prev_k) and _same(vA, prev_v)

    host, dev = SV.Shadow(sc), SV.Shadow(sc, "cuda")
    child = next(r for r in reqs if r.parent is not None)
    merges = 0
    for ev in events:
        if ev[0] == "admit":
            host.admit(ev[1], ev[3], ev[4])
            dev.admit(ev[1], ev[3], ev[4])
            continue
        if ev[0] == "free":
            _poison([kA, vA, kB, vB, prev_k, prev_v], list(ev[1]), dt)
            continue
        call = ev
        what = f"{SV.name(sc)} step {call.step} {call.kind} slots {call.slots}"
        tab.copy_(torch.tensor(call.table, dtype=torch.int32))
        lens.copy_(torch.tensor(call.lens, dtype=torch.int32))
        q, k, v = tokens.call_inputs(sc, call, idle=gen)
        decode = call.kind == "decode"
        if decode:
            for x, y in ((qd, q), (kd, k), (vd, v)):
                x.copy_(y)
            graph.replay()
            qx, kx, vx, tr, lr = qd, kd, vd, tab, lens
            oA, lA, nA = od, lsed, lens_out
            nsplit = dsplit
        else:
            b = call.slots[0]
            qx, kx, vx = q.cuda(), k.cuda(), v.cuda()
            tr, lr = tab[b:b + 1], lens[b:b + 1]
            oA, lA = torch.empty_like(qx), torch.empty(1, H, call.n_new, device="cuda")
            nA = flash_attn.fmha_fwd_kvcache(qx, kA, vA, oA, kx, vx, lr, block_table=tr, causal=True, lse=lA,
                                             num_splits=sc.num_splits, **rot, **scales)
            nsplit = SV.splits(sc, 1, call.n_new, sms)
        # pool B: the hand-written sequence
        nB = torch.empty_like(lr)
        qB = torch.empty_like(qx) if cos is not None else qx
        flash_attn.kvcache_append(kx, vx, kB, vB, lr, block_table=tr, q=qx if cos is not None else None,
                                  q_out=qB if cos is not None else None, seqlens_out=nB, **rot, **scales)
        oB, lB = torch.empty_like(oA), torch.empty_like(lA)
        flash_attn.fmha_fwd(qB, kB, vB, oB, lse=lB, causal=not decode, num_splits=sc.num_splits, seqlens_k=nB,
                            block_table=tr, **scales)
        if e4m3:
            flash_attn.kvcache_append(kx, vx, kC, vC, lr, block_table=tr, **rot)
        torch.cuda.synchronize()
        # 1. A against B
        assert _same(oA, oB) and _same(lA, lB) and torch.equal(nA, nB), f"{what}: pools A and B disagree on O / lse"
        assert _same(kA, kB) and _same(vA, vB), f"{what}: pools A and B differ"
        got = nA.cpu().tolist()
        _ok(SV.check_lengths(sc, call, [got[b] for b in call.slots] if decode else got))
        if decode:
            assert all(got[b] == 1 for b in range(B) if b not in call.slots), f"{what}: idle lengths {got}"
        # 2. written rows, q, and nothing else
        ws = SV.writes(sc, call)
        _ok(SV.check_unchanged(prev_k, kA, ws))
        _ok(SV.check_unchanged(prev_v, vA, ws))
        idx = torch.tensor([w[3] for w in ws], dtype=torch.int64, device="cuda")
        kr, vr = kA.view(-1, Hkv, D)[idx].cpu(), vA.view(-1, Hkv, D)[idx].cpu()
        t_rows = kC.view(-1, Hkv, D)[idx].cpu() if e4m3 else None
        rids = dict(zip(call.slots, call.rids))
        _ok(SV.check_written(sc, ws, tokens, rids, kr, vr, cos, sin, t_rows))
        q_rot = qB.cpu()
        _ok(SV.check_q(sc, call, tokens, q_rot, cos, sin))
        # 3. every live request's pages against its history
        host.record(ws, SV.raw(kr), SV.raw(vr))
        dev.record(ws, SV.raw(kr), SV.raw(vr))
        _ok(SV.check_history(sc, kA, vA, tab, SV.history_lens(sc, call), dev))
        # 4. O and lse against fp64
        lq, lk, hk, hv = SV.call_references(sc, call, host)
        rows = list(call.slots) if decode else [0]
        o_h, l_h = oA.cpu(), lA.cpu()
        err = SV.check_attention(sc, o_h[rows], l_h[rows], q_rot[rows], hk, hv, not decode, nsplit, lq, lk, ratios)
        assert err is None, f"{what}: {err}"
        if decode:
            idle = [b for b in range(B) if b not in call.slots]
            assert bool((o_h[idle] == 0).all()), f"{what}: O of an idle slot is not 0"
        # 5. prefill through varlen equals the unsplit paged call
        if not decode and not e4m3:
            ou, lu = oA, lA
            if nsplit > 1:
                ou, lu = torch.empty_like(oA), torch.empty_like(lA)
                flash_attn.fmha_fwd(qB, kB, vB, ou, lse=lu, causal=True, num_splits=1, seqlens_k=nB, block_table=tr)
            n = call.n_new
            qt = qB[0].transpose(0, 1).contiguous()
            ot = torch.empty_like(qt)
            lt = torch.empty(H, n, device="cuda")
            cu = torch.tensor([0, n], dtype=torch.int32, device="cuda")
            flash_attn.fmha_varlen_fwd(qt, kB, vB, ot, cu, None, n, cap, causal=True, lse=lt, block_table=tr,
                                       seqused_k=nB)
            torch.cuda.synchronize()
            assert _same(ot, ou[0].transpose(0, 1).contiguous()) and _same(lt, lu[0].contiguous()), \
                f"{what}: varlen differs from the paged call"
        # 6. the shared prefix, merged
        if decode and child.rid in call.rids and merges < MERGE_STEPS:
            b = call.slots[call.rids.index(child.rid)]
            L = SV.after_lens(sc, call)[call.slots.index(b)]
            if L > child.S:
                merges += 1
                _merge_check(sc, ratios, what, qB[b:b + 1], kB, vB, tab[b:b + 1], child.S, L, hk[rows.index(b)],
                             hv[rows.index(b)], q_rot[b:b + 1])
        prev_k.copy_(kA)
        prev_v.copy_(vA)
    assert merges == MERGE_STEPS


def _merge_check(sc, ratios, what, qc, kB, vB, row, S_, L, hk, hv, q_host):
    """Attention of one decode row over the prefix pages and over the rest (a shifted table), merged."""
    H, D, mp, ps = sc.H, sc.D, sc.max_pages, sc.page_size
    n = S_ // ps
    shifted = torch.full((1, mp), -1, dtype=torch.int32, device="cuda")
    shifted[0, :mp - n] = row[0, n:]
    parts = []
    for tbl, lk in ((row, S_), (shifted, L - S_)):
        o = torch.empty_like(qc)
        lse = torch.empty(1, H, 1, device="cuda")
        flash_attn.fmha_fwd(qc, kB, vB, o, lse=lse, seqlens_k=torch.tensor([lk], dtype=torch.int32, device="cuda"),
                            block_table=tbl, k_scale=sc.k_scale, v_scale=sc.v_scale)
        parts.append((o[:, :, 0].contiguous(), lse.view(H, 1)))
    out = torch.empty(1, H, D, dtype=qc.dtype, device="cuda")
    out_lse = torch.empty(H, 1, device="cuda")
    merge_attn_states_cuda(out, parts[0][0], parts[0][1], parts[1][0], parts[1][1], out_lse)
    torch.cuda.synchronize()
    (po, pl), (so, sl) = ((o.cpu(), l.cpu()) for o, l in parts)
    # each part against the fp64 attention over its keys
    for (o, l), keys in (((po, pl), slice(0, S_)), ((so, sl), slice(S_, L))):
        err = SV.check_attention(sc, o[:, :, None], l.view(1, H, 1), q_host, hk[None, :, keys], hv[None, :, keys],
                                 False, 1, [1], [keys.stop - keys.start])
        assert err is None, f"{what}: merge part over keys {keys}: {err}"
    ref = MR.reference(po, pl, so, sl)
    for nm, got, want, bound in (("merge O", out.cpu().double(), ref["o"], MR.o_bound(ref)),
                                 ("merge lse", out_lse.cpu().double(), ref["lse"], MR.lse_bound(ref))):
        err = (got - want).abs()
        r = float((err / bound).max())
        ratios[nm] = max(ratios.get(nm, 0.0), r)
        assert bool((err <= bound).all()), f"{what}: {nm} |err| / bound {r:.3g}"
