"""KV-cache append (flash_attn.kvcache_append, b200_kvcache_append_*) and the one-call decode step
(flash_attn.fmha_fwd_kvcache) on the GPU.

Every case of kvcache_ref.CASES runs once.  Caches, q_out and seqlens_out sit inside NaN-sentinel guard bands, caches
start with random bits, paged tables hold -1 and >= num_pages entries ("bad") or only valid ones ("good"), and the lengths
include negative ones, overflows and sequences past capacity.  Checked: every byte the append does not own comes back
unchanged (other rows, other pages, guards, k, v, q when not in place, tables, lengths); touched rows bit for bit the
restatement without rotary and within kvcache_ref.bound with it; an e4m3 append bit for bit the quantisation of the T
append on the same inputs; q_out; seqlens_out; one launch.  Then fmha_fwd_kvcache against the hand sequence and the fp64
attention references, an 8-step decode loop against a full-history fp64 reference, CUDA graph replay with new lengths,
kernel names and copies under torch.profiler in a child process, a pool past 2^31 elements written at its far end,
and every shape of tools/bench_kvcache.py at full size.
"""
import json
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

import attn_bf16_ref as BF
import attn_fp8kv_ref as F
import attn_ref as R
import attn_seqlens_ref as S
import kvcache_ref as K
from leetcuda_b200 import _capi, flash_attn

pytestmark = pytest.mark.gpu

MARGIN = 4096
SENT = {torch.float16: 0x7E01, torch.bfloat16: 0x7FC1, torch.float8_e4m3fn: 0x7F, torch.int32: -0x5A5A5A5B}
HKV, G = 2, 2


def _guarded(shape, dtype, fill=None, gen=None):
    """(buffer, view) with `MARGIN` sentinel elements either side; the view holds random bits (or `fill`)."""
    n = int(np.prod(shape))
    raw = {torch.float8_e4m3fn: torch.uint8, torch.int32: torch.int32}.get(dtype, torch.int16)
    buf = torch.empty(n + 2 * MARGIN, dtype=dtype, device="cuda")
    buf.view(raw).fill_(SENT[dtype])
    view = buf[MARGIN:MARGIN + n].view(shape)
    if fill is not None:
        view.copy_(fill)
    elif gen is not None:
        lo, hi = (0, 256) if raw == torch.uint8 else (-32768, 32768)
        view.view(raw).copy_(torch.randint(lo, hi, shape, generator=gen, dtype=torch.int64).to(raw))
    return buf, view


def _margins_ok(buf, what):
    raw = {torch.float8_e4m3fn: torch.uint8, torch.int32: torch.int32}.get(buf.dtype, torch.int16)
    bits = buf.view(raw)
    assert bool((bits[:MARGIN] == SENT[buf.dtype]).all()), f"{what}: store before the buffer"
    assert bool((bits[-MARGIN:] == SENT[buf.dtype]).all()), f"{what}: store past the buffer"


def _bits(x):
    return x.view(torch.uint8) if x.dtype == torch.float8_e4m3fn else x.view(torch.int16)


def _table(kind, B, max_pages, num_pages, gen):
    perm = torch.randperm(num_pages, generator=gen)
    table = perm[:B * max_pages].view(B, max_pages).int().clone()
    if kind == "bad":
        table.view(-1)[1::3] = -1
        table.view(-1)[2::5] = num_pages + torch.arange(table.view(-1)[2::5].numel(), dtype=torch.int32)
    return table


def _inputs(c, seed):
    gen = torch.Generator().manual_seed(seed)
    T = K.TORCH[c.T]
    B, n_new, D = len(c.lens), c.n_new, c.D
    k = torch.randn(B, HKV, n_new, D, generator=gen).to(T)
    v = torch.randn(B, HKV, n_new, D, generator=gen).to(T)
    q = torch.randn(B, HKV * G, n_new, D, generator=gen).to(T)
    rd = K.rotary_dim(c)
    cos, sin = K.tables(K.CAPACITY + n_new, rd) if rd else (None, None)
    if c.layout == "paged":
        mp = K.CAPACITY // c.page_size
        num_pages = B * mp + 3
        table = _table(c.table_kind, B, mp, num_pages, gen)
        shape, geo = (num_pages, c.page_size, HKV, D), dict(table=table, page_size=c.page_size, num_pages=num_pages)
    else:
        table, shape, geo = None, (B, HKV, K.CAPACITY, D), {}
    return gen, k, v, q, cos, sin, table, shape, geo


def _append(c, k, v, q, cos, sin, table, shape, cache_dtype, gen, scales, in_place):
    """Run kvcache_append into guarded caches; returns everything the checks need."""
    cuda = lambda x: None if x is None else x.cuda()   # noqa: E731
    kb, kc = _guarded(shape, cache_dtype, gen=gen)
    vb, vc = _guarded(shape, cache_dtype, gen=gen)
    k_before, v_before = kc.clone(), vc.clone()
    lens = torch.tensor(c.lens, dtype=torch.int32, device="cuda")
    sb, so = _guarded((len(c.lens),), torch.int32)
    kd, vd, qd = k.cuda(), v.cuda(), q.cuda()
    qob, qo = (None, qd) if in_place else _guarded(tuple(q.shape), q.dtype)
    cd, sd, td = cuda(cos), cuda(sin), cuda(table)
    torch.cuda.synchronize()
    n0 = _capi.launch_count()
    flash_attn.kvcache_append(kd, vd, kc, vc, lens, block_table=td, q=qd, q_out=qo, rotary_cos=cd, rotary_sin=sd,
                              rotary_interleaved=c.rotary == "interleaved", k_scale=scales[0], v_scale=scales[1],
                              seqlens_out=so)
    torch.cuda.synchronize()
    assert _capi.launch_count() - n0 == 1
    for buf, what in ((kb, "k_cache"), (vb, "v_cache"), (sb, "seqlens_out")) + (((qob, "q_out"),) if qob is not None
                                                                                 else ()):
        _margins_ok(buf, what)
    assert torch.equal(kd.cpu(), k) and torch.equal(vd.cpu(), v), "k / v changed"
    if not in_place:
        assert torch.equal(qd.cpu(), q), "q changed"
    assert lens.cpu().tolist() == c.lens and (td is None or torch.equal(td.cpu(), table))
    assert (cd is None or torch.equal(cd.cpu(), cos)) and (sd is None or torch.equal(sd.cpu(), sin))
    return kc.cpu(), vc.cpu(), k_before.cpu(), v_before.cpu(), qo.cpu(), so.cpu()


@pytest.mark.parametrize("i", range(len(K.CASES)))
def test_case(i):
    c = K.CASES[i]
    gen, k, v, q, cos, sin, table, shape, geo = _inputs(c, 100 + i)
    T = K.TORCH[c.T]
    rd = K.rotary_dim(c)
    inter = c.rotary == "interleaved"
    e4m3 = c.cache == "e4m3"
    scales = (0.37, 2.0) if e4m3 else (1.0, 1.0)
    dt = torch.float8_e4m3fn if e4m3 else T
    kc, vc, kb, vb, qo, so = _append(c, k, v, q, cos, sin, table, shape, dt, gen, scales, in_place=i % 2 == 1)
    B, D = len(c.lens), c.D
    flat = lambda x: x.view(-1, D)   # noqa: E731
    for after, before, new, sc, rot in ((kc, kb, k, scales[0], True), (vc, vb, v, scales[1], False)):
        err = K.check_append(flat(after), flat(before), new, c.lens, K.CAPACITY, cos, sin, rd, inter, c.T, sc,
                             rotate=rot, **geo)
        assert err is None, f"{'k' if rot else 'v'}: {err}"
    assert so.tolist() == K.seqlens_out(c.lens, c.n_new, K.CAPACITY)
    pos = K.positions(B, HKV * G, c.n_new, c.lens, K.CAPACITY)
    exact, mag = K.rotate_exact(q.reshape(-1, D), cos, sin, pos, rd, inter)
    if rd:
        assert bool(K.within(qo.reshape(-1, D), exact, mag, c.T).all()), "q_out outside the rotary bound"
    else:
        assert torch.equal(_bits(qo), _bits(q)), "q_out is not q"
    if e4m3:   # the same append into a T cache, quantised, is the e4m3 append bit for bit
        kt, vt, _, _, _, _ = _append(c, k, v, q, cos, sin, table, shape, T, gen, (1.0, 1.0), in_place=False)
        src, dst = K.cache_rows(B, HKV, c.n_new, c.lens, K.CAPACITY, geo.get("table"), geo.get("page_size"),
                                geo.get("num_pages"))
        for e, t, sc in ((kc, kt, scales[0]), (vc, vt, scales[1])):
            assert torch.equal(_bits(flat(e)[dst]), _bits(K.quantise(flat(t)[dst], sc)))


# ------------------------------------------------------------------ fmha_fwd_kvcache
def _attn_check(T, cache_dtype, o, q_rot, kcache, vcache, lens, causal, scales, what):
    """O against the fp64 reference over the cache the call attended (rows < lens), with the existing bounds."""
    D = q_rot.shape[-1]
    sc = R.kernel_scale(D)
    lq = [q_rot.shape[2]] * q_rot.shape[0]
    poly = D <= 128
    if cache_dtype == torch.float8_e4m3fn:
        kd, vd = F.decode(kcache.view(torch.uint8)), F.decode(vcache.view(torch.uint8))
        folded = float(np.float32(np.float32(sc) * np.float32(scales[0])))
        xmax = F.score_max(q_rot.double(), kd.repeat_interleave(q_rot.shape[1] // kd.shape[1], 1), folded)
        ref = S.reference(q_rot, kd, vd, folded, causal, lq, lens)
        truth = S.reference(q_rot, kd, vd, sc * scales[0], causal, lq, lens)
        want, ob = scales[1] * truth["o"], F.o_bound(ref, poly, "half" if T == torch.float16 else "bf16", scales[1], xmax)
    else:
        ref = S.reference(q_rot, kcache, vcache, sc, causal, lq, lens)
        want, ob = ref["o"], (R.o_bound(ref, poly) if T == torch.float16 else BF.o_bound(ref, poly))[1]
    err = (o.double() - want).abs()
    assert bool((err <= ob).all()), f"{what}: |err| / bound {float((err / ob).max()):.3g}"


def _dense_cache(T, dt, B, Hkv, Nk, D, gen, lens):
    k = torch.randn(B, Hkv, Nk, D, generator=gen)
    v = torch.randn(B, Hkv, Nk, D, generator=gen)
    if dt == torch.float8_e4m3fn:
        return K.quantise(k.to(T), 0.5).cuda(), K.quantise(v.to(T), 0.5).cuda()
    return k.to(T).cuda(), v.to(T).cuda()


def _to_pool(x, perm, ps):
    """[B, Hkv, Nk, D] as a pool of ps-key pages: page j of sequence b is pool page perm[b * (Nk / ps) + j]."""
    B, Hkv, Nk, D = x.shape
    bits = _bits(x).reshape(B, Hkv, Nk // ps, ps, D).permute(0, 2, 3, 1, 4).reshape(-1, ps, Hkv, D)
    out = torch.empty_like(bits)
    out[perm] = bits
    return out.view(x.dtype)


def _from_pool(pool, table):
    """The pool gathered back to [B, Hkv, Nk, D] through the table."""
    B, mp = table.shape
    _, ps, Hkv, D = pool.shape
    return _bits(pool)[table.long()].reshape(B, mp * ps, Hkv, D).transpose(1, 2).contiguous().view(pool.dtype)


KV_STEPS = [  # (T, cache, layout, rotary, n_new, causal, num_splits)
    ("half", "T", "paged", "neox", 1, False, 1),
    ("bf16", "T", "dense", "interleaved", 4, True, 1),
    ("half", "e4m3", "paged", "neox", 4, True, 2),
    ("bf16", "e4m3", "dense", "none", 1, False, 1),
]


@pytest.mark.parametrize("j", range(len(KV_STEPS)))
def test_fmha_fwd_kvcache(j):
    Tn, cache, layout, rot, n_new, causal, splits = KV_STEPS[j]
    T = K.TORCH[Tn]
    dt = torch.float8_e4m3fn if cache == "e4m3" else T
    scales = (0.5, 0.5) if cache == "e4m3" else (1.0, 1.0)
    gen = torch.Generator().manual_seed(300 + j)
    B, H, D, Nk = 4, 8, 128, 512
    lens = [0, 100, 300, 511 - n_new]
    kc, vc = _dense_cache(T, dt, B, HKV, Nk, D, gen, lens)
    table = None
    if layout == "paged":   # the same keys in 16-key pages
        ps, mp = 16, Nk // 16
        perm = torch.randperm(B * mp, generator=gen)
        table = perm.view(B, mp).int().cuda()
        kc, vc = _to_pool(kc, perm.cuda(), ps), _to_pool(vc, perm.cuda(), ps)
    q = torch.randn(B, H, n_new, D, generator=gen).to(T).cuda()
    k = torch.randn(B, HKV, n_new, D, generator=gen).to(T).cuda()
    v = torch.randn(B, HKV, n_new, D, generator=gen).to(T).cuda()
    rd = 0 if rot == "none" else D
    cos, sin = (x.cuda() for x in K.tables(Nk + n_new, rd)) if rd else (None, None)
    kw = dict(rotary_cos=cos, rotary_sin=sin, rotary_interleaved=rot == "interleaved", k_scale=scales[0],
              v_scale=scales[1])
    cl = torch.tensor(lens, dtype=torch.int32, device="cuda")
    # the hand sequence on copies
    k2, v2, q2 = kc.clone(), vc.clone(), q.clone() if rd else q
    lens2 = torch.empty_like(cl)
    flash_attn.kvcache_append(k, v, k2, v2, cl, block_table=table, q=q2 if rd else None, seqlens_out=lens2, **kw)
    o2 = torch.empty_like(q)
    fkw = dict(causal=causal, num_splits=splits, seqlens_k=lens2, block_table=table)
    if cache == "e4m3":
        fkw.update(k_scale=scales[0], v_scale=scales[1])
    flash_attn.fmha_fwd(q2, k2, v2, o2, **fkw)
    # the one call
    o = torch.empty_like(q)
    torch.cuda.synchronize()
    n0 = _capi.launch_count()
    new_lens = flash_attn.fmha_fwd_kvcache(q, kc, vc, o, k, v, cl, block_table=table, causal=causal,
                                           num_splits=splits, **kw)
    torch.cuda.synchronize()
    assert _capi.launch_count() - n0 == 1 + (2 if splits > 1 else 1)
    assert new_lens.tolist() == K.seqlens_out(lens, n_new, Nk)
    assert torch.equal(_bits(o), _bits(o2)) and torch.equal(_bits(kc), _bits(k2)) and torch.equal(_bits(vc), _bits(v2))
    # fp64: the attention over the appended cache (gathered back to dense for the paged layout)
    if layout == "paged":
        kc, vc = _from_pool(kc, table), _from_pool(vc, table)
    if splits == 1:
        _attn_check(T, dt, o, q2, kc, vc, new_lens.tolist(), causal, scales, f"kvcache step {j}")


def test_decode_loop_against_full_history():
    """8 decode steps (fp16 dense cache, NeoX rotary, B 3 at different lengths): the cache after every step holds the
    full history rotated at its positions (within the rotary bound), and O is the fp64 attention over the exact rotated
    history within attn_ref's bound plus the effect of the rotary roundings on the scores."""
    gen = torch.Generator().manual_seed(5)
    B, H, D, Nk, steps = 3, 4, 64, 64, 8
    start = [0, 5, 40]
    cos, sin = K.tables(Nk + 1, D)
    kc = torch.zeros(B, HKV, Nk, D, dtype=torch.float16, device="cuda")
    vc = torch.zeros_like(kc)
    hist_k = torch.randn(B, HKV, Nk, D, generator=gen).half()
    hist_v = torch.randn(B, HKV, Nk, D, generator=gen).half()
    # the history before the loop, rotated exactly and rounded once (what earlier appends stored)
    lens = torch.tensor(start, dtype=torch.int32, device="cuda")
    pos_all = torch.arange(Nk)
    ex_k, mag_k = K.rotate_exact(hist_k.reshape(-1, D), cos, sin, pos_all.repeat(B * HKV), D, False)
    for b in range(B):
        kc[b, :, :start[b]] = ex_k.view(B, HKV, Nk, D)[b, :, :start[b]].half().cuda()
        vc[b, :, :start[b]] = hist_v[b, :, :start[b]].cuda()
    sc = R.kernel_scale(D)
    L = list(start)
    for step in range(steps):
        q = torch.randn(B, H, 1, D, generator=gen).half()
        k = torch.stack([hist_k[b, :, L[b]:L[b] + 1] for b in range(B)])
        v = torch.stack([hist_v[b, :, L[b]:L[b] + 1] for b in range(B)])
        o = torch.empty(B, H, 1, D, dtype=torch.float16, device="cuda")
        lens = flash_attn.fmha_fwd_kvcache(q.cuda(), kc, vc, o, k.cuda(), v.cuda(), lens, rotary_cos=cos.cuda(),
                                           rotary_sin=sin.cuda())
        L = [x + 1 for x in L]
        assert lens.tolist() == L
        got_k = kc.cpu()
        for b in range(B):
            rows = slice(0, L[b])
            e = ex_k.view(B, HKV, Nk, D)[b, :, rows]
            m = mag_k.view(B, HKV, Nk, D)[b, :, rows]
            assert bool(K.within(got_k[b, :, rows], e, m, "half").all()), f"step {step}: cache of sequence {b}"
        qpos = torch.tensor([L[b] - 1 for b in range(B)]).repeat_interleave(H)
        eq, mq = K.rotate_exact(q.reshape(-1, D), cos, sin, qpos, D, False)
        eq = eq.view(B, H, 1, D)
        ref = S.reference(eq, ex_k.view(B, HKV, Nk, D), hist_v.double(), sc, False, [1] * B, L)
        # score perturbation from the roundings of q and k: |ds| <= sc (|dq| . |k| + |q| . |dk|)
        bq = K.bound(eq.reshape(-1, D), mq, "half").view(B, H, 1, D)
        bk = K.bound(ex_k, mag_k, "half").view(B, HKV, Nk, D)
        kk = ex_k.view(B, HKV, Nk, D).abs().repeat_interleave(G, 1)
        ds = sc * (bq @ kk.transpose(-1, -2) + eq.abs() @ bk.repeat_interleave(G, 1).transpose(-1, -2))
        delta = torch.stack([ds[b, :, :, :L[b]].amax(-1) for b in range(B)])
        # every weight moves by a factor within exp(+-2 delta): O by expm1(2 delta) (sigma + |O|), attn_ref's form
        ob = R.o_bound(ref, True)[1] + torch.expm1(2 * delta)[..., None] * (ref["sigma"] + ref["o"].abs())
        err = (o.cpu().double() - ref["o"]).abs()
        assert bool((err <= ob).all()), f"step {step}: |err| / bound {float((err / ob).max()):.3g}"


def test_graph_replay_with_new_lengths():
    """fmha_fwd_kvcache captured once and replayed over 4 steps with new cache_seqlens and new k, v written into the
    captured tensors: O, the caches and the lengths equal the eager call on a copy, bit for bit."""
    gen = torch.Generator().manual_seed(9)
    B, H, D, ps, mp = 4, 8, 128, 16, 8
    num_pages = B * mp
    table = torch.randperm(num_pages, generator=gen).view(B, mp).int().cuda()
    kc = torch.randn(num_pages, ps, HKV, D, generator=gen).half().cuda()
    vc = torch.randn(num_pages, ps, HKV, D, generator=gen).half().cuda()
    cos, sin = (x.cuda() for x in K.tables(mp * ps + 1, D))
    q, k, v = (torch.zeros(B, h, 1, D, dtype=torch.float16, device="cuda") for h in (H, HKV, HKV))
    o = torch.empty_like(q)
    cl = torch.zeros(B, dtype=torch.int32, device="cuda")
    kw = dict(block_table=table, rotary_cos=cos, rotary_sin=sin)
    ke, ve = kc.clone(), vc.clone()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        flash_attn.fmha_fwd_kvcache(q, kc.clone(), vc.clone(), o, k, v, cl, **kw)   # warm-up on scratch copies
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        lens_out = flash_attn.fmha_fwd_kvcache(q, kc, vc, o, k, v, cl, **kw)
    lens = [3, 17, 60, 127]
    for step in range(4):
        for x in (q, k, v):
            x.copy_(torch.randn(x.shape, generator=gen).half())
        cl.copy_(torch.tensor(lens, dtype=torch.int32))
        graph.replay()
        oe = torch.empty_like(o)
        le = flash_attn.fmha_fwd_kvcache(q, ke, ve, oe, k, v, cl.clone(), **kw)
        torch.cuda.synchronize()
        assert torch.equal(_bits(o), _bits(oe)) and torch.equal(_bits(kc), _bits(ke)) and torch.equal(_bits(vc),
                                                                                                      _bits(ve))
        assert lens_out.tolist() == le.tolist() == [min(x + 1, mp * ps) for x in lens]
        lens = [x + 1 for x in lens]


def test_kernel_names_and_no_host_copy():
    """In a child process under torch.profiler: every restated instantiation appears by its demangled name, and a
    fmha_fwd_kvcache step makes no device-to-host copy."""
    script = r"""
import json, sys, torch
sys.path.insert(0, "tests")
import kvcache_ref as K
from leetcuda_b200 import flash_attn
from torch.profiler import profile, ProfilerActivity
def run(T, e4m3):
    t = K.TORCH[T]
    dt = torch.float8_e4m3fn if e4m3 else t
    kc = torch.zeros(2, 2, 64, 64, device="cuda").to(dt); vc = kc.clone()
    q = torch.randn(2, 4, 1, 64, device="cuda").to(t); k = torch.randn(2, 2, 1, 64, device="cuda").to(t)
    cos, sin = (x.cuda() for x in K.tables(65, 64))
    flash_attn.fmha_fwd_kvcache(q, kc, vc, torch.empty_like(q), k, k.clone(), torch.tensor([3, 9], dtype=torch.int32,
                                device="cuda"), rotary_cos=cos, rotary_sin=sin)
for T in K.TYPES:
    for e in (False, True):
        run(T, e)
torch.cuda.synchronize()
with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
    for T in K.TYPES:
        for e in (False, True):
            run(T, e)
    torch.cuda.synchronize()
names = sorted({e.name for e in prof.events()})
print(json.dumps(names))
"""
    root = Path(__file__).resolve().parent.parent
    r = subprocess.run([sys.executable, "-c", script], cwd=root, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    names = json.loads(r.stdout.strip().splitlines()[-1])
    for inst in K.INSTANTIATIONS:
        assert any(K.name(inst) in n for n in names), (K.name(inst), [n for n in names if "kvcache" in n])
    assert not any("DtoH" in n or "Device -> Host" in n for n in names), [n for n in names if "DtoH" in n]


def test_pool_past_2_31_elements():
    """A paged fp16 pool of 2^31 + 2^20 elements per cache: a token written into the pool's last page (element offsets
    past 2^31) lands there, and the rows around it keep their sentinel."""
    Hkv, D, ps = 8, 128, 16
    num_pages = (2 ** 31 + 2 ** 20) // (ps * Hkv * D)
    free = torch.cuda.mem_get_info()[0]
    need = 2 * num_pages * ps * Hkv * D * 2
    if free < need + 2 ** 30:
        pytest.skip(f"needs {need / 2 ** 30:.1f} GiB free, {free / 2 ** 30:.1f} GiB available")
    kc = torch.empty(num_pages, ps, Hkv, D, dtype=torch.float16, device="cuda")
    vc = torch.empty_like(kc)
    kc.view(torch.int16)[-2:].fill_(SENT[torch.float16])
    vc.view(torch.int16)[-2:].fill_(SENT[torch.float16])
    B, n_new = 2, 3
    table = torch.tensor([[num_pages - 2, num_pages - 1], [num_pages - 1, num_pages - 2]], dtype=torch.int32,
                         device="cuda")
    lens = torch.tensor([ps - 1, ps - 2], dtype=torch.int32, device="cuda")   # both straddle into their second page
    gen = torch.Generator().manual_seed(11)
    k = torch.randn(B, Hkv, n_new, D, generator=gen).half()
    v = torch.randn(B, Hkv, n_new, D, generator=gen).half()
    flash_attn.kvcache_append(k.cuda(), v.cuda(), kc, vc, lens, block_table=table)
    torch.cuda.synchronize()
    tail_k, tail_v = kc[-2:].cpu(), vc[-2:].cpu()
    before = torch.full_like(tail_k.view(torch.int16), SENT[torch.float16]).view(torch.float16)
    geo = dict(table=[[0, 1], [1, 0]], page_size=ps, num_pages=2)
    for after, new in ((tail_k, k), (tail_v, v)):
        err = K.check_append(after.view(-1, D), before.view(-1, D), new, [ps - 1, ps - 2], 2 * ps, None, None, 0,
                             False, "half", rotate=False, **geo)
        assert err is None, err
    assert (num_pages - 1) * ps * Hkv * D >= 2 ** 31
    del kc, vc
    torch.cuda.empty_cache()


# ------------------------------------------------------------------ the benchmarked shapes
@pytest.mark.parametrize("index", range(len(K.BENCH_DECODE)))
def test_bench_decode_shape(index):
    """A decode step of tools/bench_kvcache.py at full size: fmha_fwd_kvcache equals the hand sequence bit for bit and
    the appended rows pass the restatement."""
    name, B, H, Hkv, D, n_new, ps, cache = K.BENCH_DECODE[index]
    lk = [min(x, 8192 - n_new) for x in K.bench_lengths(B, index)]   # as the tool does
    dt = torch.float8_e4m3fn if cache == "e4m3" else torch.float16
    mp = 8192 // ps
    num_pages = B * mp
    gen = torch.Generator().manual_seed(index)
    table = torch.randperm(num_pages, generator=gen).view(B, mp).int()
    kc = torch.randn(num_pages, ps, Hkv, D, device="cuda").to(dt)
    vc = torch.randn(num_pages, ps, Hkv, D, device="cuda").to(dt)
    cos, sin = K.tables(mp * ps + n_new, D)
    q = torch.randn(B, H, n_new, D, generator=gen).half()
    k = torch.randn(B, Hkv, n_new, D, generator=gen).half()
    v = torch.randn(B, Hkv, n_new, D, generator=gen).half()
    cl = torch.tensor(lk, dtype=torch.int32, device="cuda")
    scales = (0.5, 0.5) if cache == "e4m3" else (1.0, 1.0)
    kw = dict(block_table=table.cuda(), rotary_cos=cos.cuda(), rotary_sin=sin.cuda(), k_scale=scales[0],
              v_scale=scales[1])
    k0, v0 = kc.clone(), vc.clone()
    o = torch.empty(B, H, n_new, D, dtype=torch.float16, device="cuda")
    lens = flash_attn.fmha_fwd_kvcache(q.cuda(), kc, vc, o, k.cuda(), v.cuda(), cl, num_splits=0, **kw)
    q2 = q.cuda()
    l2 = torch.empty_like(cl)
    flash_attn.kvcache_append(k.cuda(), v.cuda(), k0, v0, cl, q=q2, seqlens_out=l2, **kw)
    o2 = torch.empty_like(o)
    fkw = dict(num_splits=0, seqlens_k=l2, block_table=kw["block_table"])
    if cache == "e4m3":
        fkw.update(k_scale=scales[0], v_scale=scales[1])
    flash_attn.fmha_fwd(q2, k0, v0, o2, **fkw)
    torch.cuda.synchronize()
    assert torch.equal(_bits(o), _bits(o2)) and lens.tolist() == l2.tolist() == [x + 1 for x in lk]
    assert torch.equal(_bits(kc), _bits(k0)) and torch.equal(_bits(vc), _bits(v0))
    src, dst = K.cache_rows(B, Hkv, n_new, lk, mp * ps, table, ps, num_pages)
    exact, mag = K.rotate_exact(k.reshape(-1, D)[src], cos, sin, K.positions(B, Hkv, n_new, lk, mp * ps)[src], D, False)
    got = _bits(kc).view(-1, D)[dst.cuda()].view(dt).cpu()
    if cache == "e4m3":
        b = K.bound(exact, mag, "half")
        lo, hi = K.quantise((exact - b).half(), scales[0]).float(), K.quantise((exact + b).half(), scales[0]).float()
        assert bool(((got.float() >= torch.minimum(lo, hi)) & (got.float() <= torch.maximum(lo, hi))).all())
    else:
        assert bool(K.within(got, exact, mag, "half").all())


@pytest.mark.parametrize("index", range(len(K.BENCH_APPEND)))
def test_bench_append_shape(index):
    name, B, Hkv, D, n_new, cache = K.BENCH_APPEND[index]
    Nk = 8192 + n_new
    lk = [min(x, 8192) for x in K.bench_lengths(B, 10 + index)]
    dt = torch.float8_e4m3fn if cache == "e4m3" else torch.float16
    gen = torch.Generator().manual_seed(20 + index)
    kc = torch.randn(B, Hkv, Nk, D, device="cuda").to(dt)
    vc = torch.randn(B, Hkv, Nk, D, device="cuda").to(dt)
    kb, vb = kc.cpu(), vc.cpu()
    k = torch.randn(B, Hkv, n_new, D, generator=gen).half()
    v = torch.randn(B, Hkv, n_new, D, generator=gen).half()
    cos, sin = K.tables(Nk + n_new, D)
    sc = 0.5 if cache == "e4m3" else 1.0
    flash_attn.kvcache_append(k.cuda(), v.cuda(), kc, vc, torch.tensor(lk, dtype=torch.int32, device="cuda"),
                              rotary_cos=cos.cuda(), rotary_sin=sin.cuda(), k_scale=sc, v_scale=sc)
    torch.cuda.synchronize()
    for after, before, new, rot in ((kc.cpu(), kb, k, True), (vc.cpu(), vb, v, False)):
        err = K.check_append(after.view(-1, D), before.view(-1, D), new, lk, Nk, cos, sin, D, False, "half", sc,
                             rotate=rot)
        assert err is None, err
