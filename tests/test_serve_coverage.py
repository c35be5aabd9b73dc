"""The serving schedule of serve_ref reaches what test_serve_gpu.py claims for it: the scenario table covers both element
types, T and e4m3 caches with distinct k / v scales, page sizes 16 .. 256, the three attention families and a two-slab
head dim, G = 1, 4 and MQA, every rotary layout and num_splits 0, 1 and > 1; and every scenario's schedule walks every
key length residue at a decode step, ends chunks on both sides of page and key-block edges, reuses freed pages for other
requests, appends to a shared prefix from both of its requests, overflows capacity and changes the decode batch between
graph replays."""
import pytest

import serve_ref as SV

SC = SV.SCENARIOS
MIN_REUSED = 8


def _calls(sc):
    return [e for e in SV.schedule(sc) if isinstance(e, SV.Call)]


def test_scenario_table_covers_the_serving_space():
    assert {s.T for s in SC} == {"half", "bf16"}
    assert {s.cache for s in SC} == {"T", "e4m3"}
    assert all(s.k_scale != s.v_scale for s in SC if s.cache == "e4m3")
    assert {16, 32, 64, 256} <= {s.page_size for s in SC}
    assert {"D<=64", "64<D<=128", "D>128"} <= {SV.R.family(s.D)[0] for s in SC}
    assert any(s.D > 256 for s in SC), "a head dim of more than one 256-column slab"
    assert {1, 4} <= {s.H // s.Hkv for s in SC} and any(s.Hkv == 1 for s in SC)
    assert {"neox", "gptj", "none"} <= {s.rotary for s in SC}
    assert any(0 < s.rotary_dim < s.D for s in SC), "partial rotary"
    assert {0, 1} <= {s.num_splits for s in SC} and any(s.num_splits > 1 for s in SC)
    assert len({s.seed for s in SC}) == len(SC)


@pytest.mark.parametrize("i", range(len(SC)))
def test_decode_lengths_walk_every_residue(i):
    sc = SC[i]
    lk = {x for c in _calls(sc) if c.kind == "decode" for x in SV.after_lens(sc, c)}
    kb, ps = SV.kbn(sc), sc.page_size
    assert {x % kb for x in lk} == set(range(kb)), sorted(set(range(kb)) - {x % kb for x in lk})
    want = set(range(ps)) if ps <= 64 else {0, 1, ps // 2, ps - 1}
    assert want <= {x % ps for x in lk}, sorted(want - {x % ps for x in lk})


@pytest.mark.parametrize("i", range(len(SC)))
def test_chunk_ends_straddle_page_and_block_edges(i):
    sc = SC[i]
    ends = {SV.after_lens(sc, c)[0] for c in _calls(sc) if c.kind == "prefill"}
    for m in (sc.page_size, SV.kbn(sc)):
        assert {m - 1, 0, 1} <= {e % m for e in ends}, (m, sorted(ends))
    starts = {c.lens[c.slots[0]] for c in _calls(sc) if c.kind == "prefill"}
    assert 0 in starts and any(s and s % sc.page_size == 0 for s in starts), "chunks start at 0 and on a page edge"


@pytest.mark.parametrize("i", range(len(SC)))
def test_pages_are_reused_by_other_requests(i):
    sc = SC[i]
    owners = {}
    for c in _calls(sc):
        for b, rid in zip(c.slots, c.rids):
            for p in c.table[b]:
                if p >= 0:
                    owners.setdefault(p, set()).add(rid)
    assert sum(len(o) > 1 for o in owners.values()) >= MIN_REUSED
    frees = [e for e in SV.schedule(sc) if e[0] == "free"]
    assert frees, "no page is ever freed"


@pytest.mark.parametrize("i", range(len(SC)))
def test_shared_prefix_both_append(i):
    sc = SC[i]
    reqs = SV.requests(sc)
    child = next(r for r in reqs if r.parent is not None)
    assert child.S > 0 and child.S % sc.page_size == 0
    both = [c for c in _calls(sc) if c.kind == "decode" and {child.rid, child.parent} <= set(c.rids)]
    assert both, "parent and child never decode together"
    c = both[0]
    pb, cb = (c.slots[c.rids.index(r)] for r in (child.parent, child.rid))
    n = child.S // sc.page_size
    assert c.table[pb][:n] == c.table[cb][:n] and c.table[pb][n:] != c.table[cb][n:]
    assert c.lens[pb] < SV.capacity(sc) and c.lens[cb] < SV.capacity(sc)
    # the parent finishes first: the child reads the shared pages after their first owner is gone
    last = {r: max(k for k, x in enumerate(_calls(sc)) if r in x.rids) for r in (child.parent, child.rid)}
    assert last[child.parent] < last[child.rid]


@pytest.mark.parametrize("i", range(len(SC)))
def test_a_request_overflows_capacity(i):
    sc = SC[i]
    cap = SV.capacity(sc)
    over = [c for c in _calls(sc) if c.kind == "decode" and any(c.lens[b] == cap for b in c.slots)]
    assert len(over) >= 2


@pytest.mark.parametrize("i", range(len(SC)))
def test_empty_prompt_and_idle_slots(i):
    sc = SC[i]
    reqs = SV.requests(sc)
    assert any(not r.ends and r.S == 0 for r in reqs)
    dec = [c for c in _calls(sc) if c.kind == "decode"]
    assert any(len(c.slots) < SV.B_MAX for c in dec), "no decode step with an idle slot"
    assert all(c.table[b] == [-1] * sc.max_pages and c.lens[b] == 0 for c in dec for b in range(SV.B_MAX)
               if b not in c.slots)
    assert 12 <= len(reqs) <= 16


@pytest.mark.parametrize("i", range(len(SC)))
def test_graph_replays_after_the_batch_changes(i):
    dec = [c.slots for c in _calls(SC[i]) if c.kind == "decode"]
    changes = sum(a != b for a, b in zip(dec, dec[1:]))
    assert changes >= 4 and any(len(s) == SV.B_MAX for s in dec)


def test_auto_splits_split_a_decode_step():
    auto = [s for s in SC if s.num_splits == 0]
    assert auto
    for sc in auto:
        assert SV.splits(sc, SV.B_MAX, 1, SV.H100_SMS) > 1, SV.name(sc)
