"""A paged serving schedule restated on the CPU: the scenario table, a deterministic scheduler over a reused page pool,
the host shadow of every request, the checks of a step, and a host model of a correct server (with injectable
bookkeeping mistakes) for the sharpness test.  Used by test_serve_gpu.py, test_serve_coverage.py and
test_serve_sharpness.py.

Serving.  B_MAX slots share one pool of pages [num_pages, page_size, Hkv, D].  Requests arrive, take a free slot, prefill
their prompt in chunks (one fmha_fwd_kvcache(B=1, causal=True) per chunk on their table row), then decode one token per
step in one call over all B_MAX slots, finish and give their pages back.  Pages come from a LIFO free list (a page freed
at one step is the next one handed out) and are refcounted: a request may start on whole prefix pages of a live one
(cache_seqlens = S, a multiple of page_size).  In a decode call every slot that is not decoding (idle or mid-prefill)
holds cache_seqlens = 0 and a table row of -1: its token is dropped and its one key reads zeros, so its O is 0.

Token j of a request that starts at S has position S + j; a decode token past capacity (max_pages * page_size) is
dropped and its q is rotated at capacity (kvcache_ref: positions).  The shadow of a slot holds the cache bits stored
for every position of its request, so the pool gathered through the request's table must equal it bit for bit.

Nothing here adds a bound: the rows use kvcache_ref's, the attention attn_ref / attn_bf16_ref / attn_fp8kv_ref's with
attn_split_ref's combine_bound when a call splits, and the merge merge_ref's.
"""
from __future__ import annotations

import math
from collections import namedtuple

import numpy as np
import torch

import attn_bf16_ref as BF
import attn_fp8kv_ref as F
import attn_mask_ref as M
import attn_ref as R
import attn_seqlens_ref as S
import attn_split_ref as SR
import bench_workloads as BW
import kvcache_ref as K

B_MAX = 8
H100_SMS = 132                  # SMs of an H100 SXM: the split counts the coverage test expects
POISON = {torch.float16: 0x7E01, torch.bfloat16: 0x7FC1, torch.float8_e4m3fn: 0x7F}   # NaN bits of a freed page

# rotary: "none", "neox" or "gptj" over rotary_dim columns (rotary_dim < D: partial)
Scenario = namedtuple("Scenario", "T cache page_size D H Hkv rotary rotary_dim num_splits k_scale v_scale max_pages seed")
SCENARIOS = [
    Scenario("half", "T", 16, 64, 8, 8, "neox", 64, 1, 1.0, 1.0, 32, 1),          # G 1, kBN 128
    Scenario("bf16", "T", 32, 128, 8, 2, "gptj", 128, 3, 1.0, 1.0, 16, 2),        # G 4, three splits
    Scenario("half", "e4m3", 64, 128, 8, 1, "neox", 64, 0, 0.37, 2.0, 16, 3),     # MQA, partial rotary, auto splits
    Scenario("bf16", "e4m3", 256, 256, 8, 2, "neox", 256, 2, 0.5, 1.5, 2, 4),     # D > 128, two splits
    Scenario("half", "T", 16, 320, 4, 1, "none", 0, 2, 1.0, 1.0, 24, 5),          # two slabs, MQA, no rotary
    Scenario("bf16", "T", 64, 64, 8, 2, "gptj", 32, 1, 1.0, 1.0, 8, 6),           # G 4, partial GPT-J
]


def name(sc):
    return f"{sc.T}-{sc.cache}-p{sc.page_size}-D{sc.D}-H{sc.H}/{sc.Hkv}-{sc.rotary}{sc.rotary_dim}-s{sc.num_splits}"


def kbn(sc):
    return M.kernel_shape(sc.D)[0]


def capacity(sc):
    return sc.max_pages * sc.page_size


def num_pages(sc):
    return B_MAX * sc.max_pages + 4


def dtype(sc):
    return torch.float8_e4m3fn if sc.cache == "e4m3" else K.TORCH[sc.T]


def interleaved(sc):
    return sc.rotary == "gptj"


def rotary_tables(sc):
    """fp32 cos, sin long enough for a chunk of up to capacity tokens at any position (None without rotary)."""
    return K.tables(2 * capacity(sc) + 1, sc.rotary_dim) if sc.rotary_dim else (None, None)


def splits(sc, B, Nq, sms):
    """The split count of a call: num_splits, or for 0 bench_workloads.auto_splits on the padded shape."""
    return sc.num_splits or BW.auto_splits(B, sc.H, sc.Hkv, Nq, capacity(sc), sc.D, sms)


def raw(x):
    return x.view(torch.uint8) if x.dtype == torch.float8_e4m3fn else x.view(torch.int16)


# ------------------------------------------------------------------ requests
Request = namedtuple("Request", "rid arrive parent S ends n_decode")   # ends: absolute chunk-end positions


def requests(sc):
    """About 14 requests: one with an empty prompt, one that decodes past capacity, a parent and a child that starts on
    the parent's first S positions (whole pages), and ten more whose chunk ends sit on and next to page and key-block
    edges or anywhere."""
    rng = np.random.default_rng(sc.seed)
    ps, kb, cap = sc.page_size, kbn(sc), capacity(sc)
    edges = sorted({e + d for m in (ps, kb) for e in range(m, cap, m) for d in (-1, 0, 1)} | {1})
    edges = [e for e in edges if e <= cap // 2]
    S_ = ps * max(1, min(2, (cap // 3) // ps))
    out = [Request(0, 0, None, 0, (), 40),
           Request(1, 1, None, 0, (1, kb - 1, 2 * kb, cap - 3), 10),
           Request(2, 0, None, 0, (ps - 1, S_, S_ + 1), 30),
           Request(3, None, 2, S_, (S_ + 1, S_ + kb), 45)]
    for i in range(10):
        n = int(rng.integers(1, 4))
        if i % 2 == 0:
            ends = sorted(set(int(x) for x in rng.choice(edges, size=n, replace=False)))
        else:
            ends = sorted(set(int(x) for x in rng.integers(2, cap // 2, size=n)))
        out.append(Request(4 + i, 2 + 2 * i, None, 0, tuple(ends), int(rng.integers(16, 57))))
    return out


# ------------------------------------------------------------------ the scheduler
# Events, in order:
#   ("free", pages)                         pages whose last owner finished (the pool fills them with NaN bits)
#   ("admit", slot, rid, parent_slot, S)    a request takes a slot (parent_slot: the slot it shares S positions with)
#   Call(...)                               one call of the system under test
Call = namedtuple("Call", "kind step slots rids toks lens table n_new")
# kind "prefill": slots = (slot,), n_new = the chunk; "decode": slots = every decoding slot, n_new = 1.  toks[i]: the
# request's first token index of the call; lens: the B_MAX cache_seqlens of the call; table: its B_MAX table rows
# (a decode call's non-decoding slots -1, a prefill call's true rows).  Live lengths after the call: after_lens(call).


def schedule(sc, reqs=None):
    reqs = requests(sc) if reqs is None else reqs
    ps, cap, mp, npg = sc.page_size, capacity(sc), sc.max_pages, num_pages(sc)
    free = list(range(npg))[::-1]          # LIFO: pop() hands out the page freed last
    ref = [0] * npg
    slots = [None] * B_MAX                 # per slot: dict(req, pages, L, chunk, tok, done, decoding)
    pending = list(reqs)
    events = []
    step = 0

    def ensure(st, upto):
        need = -(-min(upto, cap) // ps)
        while len(st["pages"]) < need:
            p = free.pop()
            ref[p] += 1
            st["pages"].append(p)

    def rows(decoding_only):
        t = [[-1] * mp for _ in range(B_MAX)]
        lens = [0] * B_MAX
        for b, st in enumerate(slots):
            if st is None or (decoding_only and not st["decoding"]):
                continue
            t[b][:len(st["pages"])] = st["pages"]
            lens[b] = st["L"]
        return t, lens

    while pending or any(slots):
        for r in list(pending):
            if None not in slots:
                break
            if r.parent is None:
                if r.arrive > step:
                    continue
                pslot, pages = None, []
            else:
                pslot = next((b for b, st in enumerate(slots) if st and st["req"].rid == r.parent and st["decoding"]
                              and st["L"] >= r.S), None)
                if pslot is None:
                    continue
                pages = slots[pslot]["pages"][:r.S // ps]
                for p in pages:
                    ref[p] += 1
            b = slots.index(None)
            slots[b] = dict(req=r, pages=list(pages), L=r.S, chunk=0, tok=0, done=0, decoding=not r.ends)
            pending.remove(r)
            events.append(("admit", b, r.rid, pslot, r.S))
        for b, st in enumerate(slots):    # one prefill chunk per prefilling request
            if st is None or st["decoding"]:
                continue
            r = st["req"]
            n = r.ends[st["chunk"]] - st["L"]
            ensure(st, st["L"] + n)
            t, lens = rows(False)
            events.append(Call("prefill", step, (b,), (r.rid,), (st["tok"],), lens, t, n))
            st["L"] += n
            st["tok"] += n
            st["chunk"] += 1
        dec = [b for b, st in enumerate(slots) if st is not None and st["decoding"]]
        if dec:
            for b in dec:
                ensure(slots[b], slots[b]["L"] + 1)
            t, lens = rows(True)
            events.append(Call("decode", step, tuple(dec), tuple(slots[b]["req"].rid for b in dec),
                               tuple(slots[b]["tok"] for b in dec), lens, t, 1))
            freed = []
            for b in dec:
                st = slots[b]
                st["L"] = min(st["L"] + 1, cap)
                st["tok"] += 1
                st["done"] += 1
                if st["done"] == st["req"].n_decode:
                    for p in st["pages"]:
                        ref[p] -= 1
                        if ref[p] == 0:
                            free.append(p)
                            freed.append(p)
                    slots[b] = None
            if freed:
                events.append(("free", tuple(freed)))
        for st in slots:   # a request whose prompt is done decodes from the next step on
            if st is not None and not st["decoding"] and st["chunk"] == len(st["req"].ends):
                st["decoding"] = True
        step += 1
    return events


def after_lens(sc, call):
    """Expected returned lengths of a call, per slot of the call."""
    return [min(call.lens[b] + call.n_new, capacity(sc)) for b in call.slots]


def writes(sc, call):
    """[(slot, token index, position, pool row)] of every token the call stores; pool rows index the pool viewed as
    [num_pages * page_size, Hkv, D]."""
    out = []
    cap = capacity(sc)
    for i, b in enumerate(call.slots):
        for t in range(call.n_new):
            s = K.slot(b, t, call.lens[b], cap, call.table, sc.page_size, num_pages(sc))
            if s is not None:
                out.append((b, call.toks[i] + t, call.lens[b] + t, s[0] * sc.page_size + s[1]))
    return out


def q_positions(sc, call):
    """[len(slots), n_new] absolute positions q is rotated at."""
    return [[min(call.lens[b], capacity(sc)) + t for t in range(call.n_new)] for b in call.slots]


# ------------------------------------------------------------------ tokens
class Tokens:
    """The seeded k, v [n, Hkv, D] and q [n, H, D] (T) of every request, by token index."""

    def __init__(self, sc, reqs):
        g = torch.Generator().manual_seed(1000 + sc.seed)
        T = K.TORCH[sc.T]
        self.k, self.v, self.q = {}, {}, {}
        for r in reqs:
            n = (r.ends[-1] - r.S if r.ends else 0) + r.n_decode
            self.k[r.rid] = torch.randn(n, sc.Hkv, sc.D, generator=g).to(T)
            self.v[r.rid] = torch.randn(n, sc.Hkv, sc.D, generator=g).to(T)
            self.q[r.rid] = torch.randn(n, sc.H, sc.D, generator=g).to(T)

    def call_inputs(self, sc, call, idle=None):
        """q [B, H, n, D], k, v [B, Hkv, n, D] of a call: B = 1 for a prefill, B_MAX for a decode (slots that are not in
        the call get `idle` (a generator) random tokens, or zeros)."""
        T = K.TORCH[sc.T]
        B = 1 if call.kind == "prefill" else B_MAX
        shapes = ((sc.H, call.n_new, sc.D), (sc.Hkv, call.n_new, sc.D), (sc.Hkv, call.n_new, sc.D))
        out = [torch.zeros((B,) + s, dtype=T) if idle is None else torch.randn((B,) + s, generator=idle).to(T)
               for s in shapes]
        for i, b in enumerate(call.slots):
            row = 0 if call.kind == "prefill" else b
            t0, r = call.toks[i], call.rids[i]
            for x, src in zip(out, (self.q, self.k, self.v)):
                x[row] = src[r][t0:t0 + call.n_new].transpose(0, 1)
        return out


# ------------------------------------------------------------------ the shadow
class Shadow:
    """Per slot, the cache bits stored for every position of its request: k, v [B_MAX, capacity, Hkv, D] raw (int16
    or uint8), on any device."""

    def __init__(self, sc, device="cpu"):
        rd = torch.uint8 if sc.cache == "e4m3" else torch.int16
        self.k = torch.zeros(B_MAX, capacity(sc), sc.Hkv, sc.D, dtype=rd, device=device)
        self.v = torch.zeros_like(self.k)

    def admit(self, slot, parent_slot, S_):
        if parent_slot is not None:
            self.k[slot, :S_] = self.k[parent_slot, :S_]
            self.v[slot, :S_] = self.v[parent_slot, :S_]

    def record(self, ws, k_rows, v_rows):
        """Store the rows written at ws (writes()) from k_rows, v_rows [len(ws), Hkv, D] raw."""
        if not ws:
            return
        b = torch.tensor([w[0] for w in ws], device=self.k.device)
        p = torch.tensor([w[2] for w in ws], device=self.k.device)
        self.k[b, p] = k_rows.to(self.k.device)
        self.v[b, p] = v_rows.to(self.k.device)

    def values(self, which, slots, sc):
        """fp64 values [len(slots), Hkv, capacity, D] of the shadow's k or v of some slots (positions past a length
        hold zeros or stale values: callers mask them)."""
        x = (self.k if which == "k" else self.v)[list(slots)].cpu()
        if sc.cache == "e4m3":
            x = F.decode(x)
        else:
            x = x.view(K.TORCH[sc.T]).double()
        return x.transpose(1, 2)


# ------------------------------------------------------------------ checks (each returns None or the first violation)
def check_unchanged(before, after, ws):
    """Every pool row but the written ones holds its bits (pools [num_pages, page_size, Hkv, D], any device)."""
    a = raw(after).reshape(-1, after.shape[2], after.shape[3])
    b = raw(before).reshape(a.shape)
    keep = torch.ones(a.shape[0], dtype=torch.bool, device=a.device)
    if ws:
        keep[torch.tensor([w[3] for w in ws], device=a.device)] = False
    if not torch.equal(a[keep], b[keep]):
        bad = ((a != b).flatten(1).any(1) & keep).nonzero()[:4].flatten().tolist()
        return f"pool rows changed that the call does not own: {bad}"
    return None


def check_written(sc, ws, tokens, rids, k_rows, v_rows, cos, sin, t_rows=None):
    """The rows written at ws are the request's tokens at their absolute positions: rotated k within kvcache_ref's
    rotary bound of the exact rotation, e4m3 bit for bit the quantisation of the T append's rows t_rows, everything
    else bit for bit.  k_rows, v_rows: [n, Hkv, D] cache rows (CPU) read at ws; rids: {slot: request id}."""
    if not ws:
        return None
    D, Hkv = sc.D, sc.Hkv
    kn = torch.stack([tokens.k[rids[w[0]]][w[1]] for w in ws])
    vn = torch.stack([tokens.v[rids[w[0]]][w[1]] for w in ws])
    e4m3 = sc.cache == "e4m3"
    want_v = K.quantise(vn, sc.v_scale) if e4m3 else vn
    if not torch.equal(raw(v_rows), raw(want_v)):
        return "a written v row is not the request's token"
    if sc.rotary_dim == 0:
        want_k = K.quantise(kn, sc.k_scale) if e4m3 else kn
        return None if torch.equal(raw(k_rows), raw(want_k)) else "a written k row is not the request's token"
    pos = torch.tensor([w[2] for w in ws]).repeat_interleave(Hkv)
    exact, mag = K.rotate_exact(kn.reshape(-1, D), cos, sin, pos, sc.rotary_dim, interleaved(sc))
    got = t_rows if e4m3 else k_rows
    if not bool(K.within(got.reshape(-1, D), exact, mag, sc.T).all()):
        return "a written k row is outside the rotary bound of its token at its position"
    if e4m3 and not torch.equal(raw(k_rows), raw(K.quantise(t_rows, sc.k_scale))):
        return "a written e4m3 k row is not the quantisation of the T append"
    return None


def check_q(sc, call, tokens, q_rot, cos, sin):
    """The rotated q [B, H, n, D] (CPU) of the call's slots within the rotary bound at their absolute positions."""
    if sc.rotary_dim == 0:
        return None
    for i, b in enumerate(call.slots):
        row = 0 if call.kind == "prefill" else b
        q = tokens.q[call.rids[i]][call.toks[i]:call.toks[i] + call.n_new]         # [n, H, D]
        pos = torch.tensor(q_positions(sc, call)[i]).repeat_interleave(sc.H)
        exact, mag = K.rotate_exact(q.reshape(-1, sc.D), cos, sin, pos, sc.rotary_dim, interleaved(sc))
        if not bool(K.within(q_rot[row].transpose(0, 1).reshape(-1, sc.D), exact, mag, sc.T).all()):
            return f"q of slot {b} is outside the rotary bound at its positions"
    return None


def check_history(sc, pool_k, pool_v, table, lens, shadow):
    """The pool gathered through every live slot's table row equals its shadow bit for bit at positions < its length
    (table: [B_MAX, max_pages] int tensor on the pools' device; lens: B_MAX ints)."""
    ps, cap = sc.page_size, capacity(sc)
    live = torch.arange(cap, device=table.device)[None, :] < torch.tensor(lens, device=table.device)[:, None]
    idx = table.long().clamp(min=0)
    for which, pool, sh in (("k", pool_k, shadow.k), ("v", pool_v, shadow.v)):
        g = raw(pool)[idx].reshape(B_MAX, cap, sc.Hkv, sc.D)
        ok = (g == sh).flatten(2).all(2) | ~live
        if not bool(ok.all()):
            b, p = (~ok).nonzero()[0].tolist()
            return f"{which} cache of slot {b} at position {p} is not its request's history"
    return None


def check_lengths(sc, call, got):
    want = after_lens(sc, call)
    return None if list(got) == want else f"returned lengths {list(got)}, want {want}"


def attention_bounds(sc, q, hk, hv, causal, nsplit, lq, lk):
    """(truth O, truth lse, O bound, lse bound) of rows q [B, H, Nq, D] (T, CPU) over histories hk, hv
    [B, Hkv, Nk, D] (fp64 values), with the library's per-element bounds."""
    D = sc.D
    poly = D <= 128
    sc0 = R.kernel_scale(D)
    if sc.cache == "e4m3":
        folded = float(np.float32(np.float32(sc0) * np.float32(sc.k_scale)))
        G = sc.H // sc.Hkv
        xmax = F.score_max(q.double(), SR.expand(hk, G), folded)
        truth = S.reference(q, hk, hv, sc0 * sc.k_scale, causal, lq, lk)
        if nsplit > 1:
            parts = S.part_references(q, hk, hv, folded, causal, nsplit, lq, lk)
            vmax = SR.expand(hv.abs().amax(-2, keepdim=True), G)
            _, _, _, ob, lb = F.combine_bound(parts, poly, sc.T, sc.v_scale, xmax, vmax)
        else:
            ref = S.reference(q, hk, hv, folded, causal, lq, lk)
            ob, lb = F.o_bound(ref, poly, sc.T, sc.v_scale, xmax), F.lse_bound(ref, poly, xmax)
        return sc.v_scale * truth["o"], truth["lse"], ob, lb
    mod = BF if sc.T == "bf16" else R
    if nsplit > 1:
        parts = S.part_references(q, hk, hv, sc0, causal, nsplit, lq, lk)
        o, L, _, ob, lb = (BF.combine_bound if sc.T == "bf16" else SR.combine_bound)(parts, poly)
        return o, L, ob, lb
    ref = S.reference(q, hk, hv, sc0, causal, lq, lk)
    return ref["o"], ref["lse"], mod.o_bound(ref, poly)[1], mod.lse_bound(ref, poly)


def check_attention(sc, o, lse, q, hk, hv, causal, nsplit, lq, lk, ratios=None):
    """O [B, H, Nq, D] and lse [B, H, Nq] (CPU) within the bounds of attention_bounds at every row with a visible key;
    updates ratios["O"], ratios["lse"] with the largest |err| / bound."""
    want_o, want_l, ob, lb = attention_bounds(sc, q, hk, hv, causal, nsplit, lq, lk)
    Nq = q.shape[2]
    rows = torch.stack([torch.arange(Nq) < x for x in lq])[:, None, :].expand(o.shape[:3])
    for nm, got, want, bound in (("O", o.double(), want_o, ob), ("lse", lse.double(), want_l, lb)):
        err = (got - want).abs()
        if nm == "O":
            err, bound = err[rows], bound.expand(err.shape)[rows]
        else:
            err, bound = err[rows], bound[rows]
        ratio = float(torch.nan_to_num(err / bound, nan=math.inf).max()) if err.numel() else 0.0
        if ratios is not None:
            ratios[nm] = max(ratios.get(nm, 0.0), ratio)
        if not bool((err <= bound).all()):
            return f"{nm}: |err| / bound {ratio:.3g}"
    return None


def call_references(sc, call, shadow):
    """(q rows, lq, lk, hk, hv) the fp64 reference of a call needs: the rows of its slots, histories from the shadow
    after the call (positions < the new length)."""
    new = after_lens(sc, call)
    hk, hv = shadow.values("k", call.slots, sc), shadow.values("v", call.slots, sc)
    return [call.n_new] * len(call.slots), new, hk, hv


# ------------------------------------------------------------------ a host model of the server (sharpness)
MISTAKES = ("append_early", "append_late", "stuck_length", "foreign_page", "freed_page", "drop_last_key",
            "stale_key")


def _rotate_T(sc, x, pos, cos, sin):
    """x [n, heads, D] (T) rotated exactly at positions pos [n] and rounded once to T: a correct kernel's rows."""
    n, h, D = x.shape
    if sc.rotary_dim == 0:
        return x.clone()
    exact, _ = K.rotate_exact(x.reshape(-1, D), cos, sin, torch.tensor(pos).repeat_interleave(h), sc.rotary_dim,
                              interleaved(sc))
    return exact.to(K.TORCH[sc.T]).view(n, h, D)


def host_call(sc, call, pool_k, pool_v, tokens, cos, sin, freed, mistake=None):
    """One call of a correct server on CPU pools (modified in place): the append (rotary exact, rounded to T; e4m3
    quantised), then the fp64 attention over what its table gathers, rounded to T.  Returns (O, lse, new lengths,
    q_rot, T rows of the written k).  `mistake` injects one bookkeeping error (MISTAKES); freed: pages on the free
    list."""
    ps, cap, T = sc.page_size, capacity(sc), K.TORCH[sc.T]
    table = [list(r) for r in call.table]
    lens = list(call.lens)
    if mistake == "foreign_page":   # the page of the first slot's first new token taken from another live row
        b = call.slots[0]
        others = [t[0] for c, t in enumerate(table) if c != b and t[0] >= 0]
        if lens[b] < cap and others:
            table[b][lens[b] // ps] = others[0]
    shift = {"append_early": -1, "append_late": 1}.get(mistake, 0)
    q, k, v = tokens.call_inputs(sc, call)
    t_rows = []
    flat_k, flat_v = pool_k.view(-1, sc.Hkv, sc.D), pool_v.view(-1, sc.Hkv, sc.D)
    q_rot = q.clone()
    for i, b in enumerate(call.slots):
        row = 0 if call.kind == "prefill" else b
        L = min(lens[b], cap)
        pos = [L + t for t in range(call.n_new)]
        q_rot[row] = _rotate_T(sc, q[row].transpose(0, 1), pos, cos, sin).transpose(0, 1)
        kr = _rotate_T(sc, k[row].transpose(0, 1), pos, cos, sin)
        for t, p in enumerate(pos):
            p += shift
            if not 0 <= p < cap or table[b][p // ps] < 0:
                continue
            dst = table[b][p // ps] * ps + p % ps
            if sc.cache == "e4m3":
                flat_k[dst], flat_v[dst] = K.quantise(kr[t], sc.k_scale), K.quantise(v[row, :, t], sc.v_scale)
                t_rows.append(kr[t])
            else:
                flat_k[dst], flat_v[dst] = kr[t], v[row, :, t]
    new = [min(min(lens[b], cap) + call.n_new, cap) for b in call.slots]
    if mistake == "stuck_length" and call.kind == "prefill":
        new = [min(lens[b], cap) for b in call.slots]
    lk = list(new)
    if mistake == "drop_last_key":
        lk = [max(x - 1, 0) for x in lk]
    if mistake == "stale_key":
        lk = [min(x + 1, cap) for x in lk]
    if mistake == "freed_page" and freed:
        b = call.slots[0]
        table[b][(lk[0] - 1) // ps] = freed[-1]
    # gather through the (possibly wrong) table: entries outside [0, num_pages) read zeros
    idx = torch.tensor([table[b] for b in call.slots], dtype=torch.int64)
    hist = []
    for pool in (pool_k, pool_v):
        g = pool[idx.clamp(min=0)].reshape(len(call.slots), cap, sc.Hkv, sc.D).clone()
        raw(g)[(idx < 0).repeat_interleave(ps, 1)] = 0
        raw(g)[torch.arange(cap)[None, :] >= torch.tensor(lk)[:, None]] = 0   # keys past a length are not read
        hist.append((F.decode(raw(g)) if sc.cache == "e4m3" else g.double()).transpose(1, 2))
    rows = q_rot[list(call.slots)] if call.kind == "decode" else q_rot
    lq = [call.n_new] * len(call.slots)
    causal = call.kind == "prefill"
    sc0 = R.kernel_scale(sc.D)
    ref = S.reference(rows, hist[0], hist[1], sc0 * sc.k_scale, causal, lq, lk)
    o = (sc.v_scale * ref["o"]).to(T)
    o_full = torch.zeros_like(q)
    lse_full = torch.zeros(q.shape[:3])
    if call.kind == "decode":
        o_full[list(call.slots)] = o
        lse_full[list(call.slots)] = ref["lse"].float()
    else:
        o_full, lse_full = o, ref["lse"].float()
    krows = torch.stack(t_rows) if t_rows else None
    return o_full, lse_full, new, q_rot, krows


def history_lens(sc, call):
    """The B_MAX lengths check_history compares after a call: the call's lengths with its slots advanced."""
    lens = list(call.lens)
    for b, x in zip(call.slots, after_lens(sc, call)):
        lens[b] = x
    return lens


def run_host(sc, events, mistake=None):
    """Drive the host model through `events` with `mistake` injected into every call, and run checks 2-4 (and the
    returned lengths) after each.  Returns None or the first violation as text."""
    reqs = requests(sc)
    tokens = Tokens(sc, reqs)
    cos, sin = rotary_tables(sc)
    shape = (num_pages(sc), sc.page_size, sc.Hkv, sc.D)
    dt = dtype(sc)
    pool_k, pool_v = torch.zeros(shape, dtype=dt), torch.zeros(shape, dtype=dt)
    shadow = Shadow(sc)
    freed = []
    for ev in events:
        if ev[0] == "admit":
            shadow.admit(ev[1], ev[3], ev[4])
            continue
        if ev[0] == "free":
            for p in ev[1]:
                raw(pool_k)[p] = POISON[dt]
                raw(pool_v)[p] = POISON[dt]
            freed += list(ev[1])
            continue
        call = ev
        freed = [p for p in freed if all(p not in row for row in call.table)]
        before_k, before_v = pool_k.clone(), pool_v.clone()
        o, lse, new, q_rot, t_rows = host_call(sc, call, pool_k, pool_v, tokens, cos, sin, freed, mistake)
        ws = writes(sc, call)
        idx = torch.tensor([w[3] for w in ws], dtype=torch.int64)
        kr, vr = pool_k.view(-1, sc.Hkv, sc.D)[idx], pool_v.view(-1, sc.Hkv, sc.D)[idx]
        err = (check_lengths(sc, call, new) or check_unchanged(before_k, pool_k, ws)
               or check_unchanged(before_v, pool_v, ws)
               or check_written(sc, ws, tokens, dict(zip(call.slots, call.rids)), kr, vr, cos, sin, t_rows)
               or check_q(sc, call, tokens, q_rot, cos, sin))
        if err:
            return err
        shadow.record(ws, raw(kr), raw(vr))
        err = check_history(sc, pool_k, pool_v, torch.tensor(call.table), history_lens(sc, call), shadow)
        if err:
            return err
        lq, lk, hk, hv = call_references(sc, call, shadow)
        rows = list(call.slots) if call.kind == "decode" else [0]
        nsplit = splits(sc, 1 if call.kind == "prefill" else B_MAX, call.n_new, H100_SMS)
        err = check_attention(sc, o[rows], lse[rows], q_rot[rows], hk, hv, call.kind == "prefill", nsplit, lq, lk)
        if err:
            return err
    return None
