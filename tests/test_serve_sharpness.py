"""The checks of test_serve_gpu.py are sharp enough: a host model of a correct server (rotary exact and rounded once,
e4m3 quantised, the fp64 attention over what its table gathers rounded to the element type) passes the checks of every
call of a short schedule, and each bookkeeping mistake a server can make is rejected by some check: an append one row
early or late, a length that does not advance after a prefill chunk, a table entry taken from another request, a freed
page read as live, the last key dropped, and one extra stale key read."""
import pytest

import serve_ref as SV


def _short(sc):
    """The schedule up to six calls past the first freed pages: prefills, decodes with idle slots, a shared prefix,
    and pages back on the free list."""
    ev = SV.schedule(sc)
    first_free = next(i for i, e in enumerate(ev) if e[0] == "free")
    calls = [i for i, e in enumerate(ev) if isinstance(e, SV.Call) and i > first_free]
    return ev[:calls[5] + 1]


SHORT = [SV.SCENARIOS[5], SV.SCENARIOS[2]._replace(max_pages=4)]   # a T cache and an e4m3 cache with partial rotary


@pytest.mark.parametrize("i", range(len(SHORT)))
def test_correct_server_passes(i):
    sc = SHORT[i]
    assert SV.run_host(sc, _short(sc)) is None


@pytest.mark.parametrize("mistake", SV.MISTAKES)
def test_mistake_is_rejected(mistake):
    sc = SHORT[0]
    err = SV.run_host(sc, _short(sc), mistake)
    assert err is not None, f"{mistake} passed every check"
