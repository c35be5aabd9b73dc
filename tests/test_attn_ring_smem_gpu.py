"""attn_ring_ref's restated shared memory against the launches: every row of the case tables with D > 512 (three and
four slabs, the rings that wrap) runs once under torch.profiler, and the `shared memory` its Kineto kernel record
carries (static + dynamic) is attn_ring_ref.smem_bytes of its head dim and K/V type.

The attention kernels declare no static shared memory (test_attn_ring_coverage), so the record is the dynamic shared
memory fmha_dispatch asked for.  The transpose pre-pass of the V^T rows shows what a static array adds: its record is
its 2112-byte tile.

torch.profiler runs in a child process, all rows in one session; this process never starts it.
The records are printed at the end of the module (pytest -s).
"""
import json
import os
import subprocess
import sys
import tempfile
import time
from pathlib import Path

import pytest
import torch

import attn_ring_ref as RR

pytestmark = pytest.mark.gpu

ROWS = [(kind, T, c) for kind, T, c in RR.table_rows() if c.D > 512]
TRANSPOSE_TILE = 32 * 33 * 2   # attn_capi.cu transpose_dn_to_nd_kernel: __shared__ __half tile[32][33]


def _row_id(i):
    kind, T, c = ROWS[i]
    return f"{kind}-{T}-{i}-D{c.D}"


def _row_call(i):
    """A call of row i on randn inputs."""
    from leetcuda_b200 import flash_attn
    from test_attn_gqa_gpu import _inputs
    from test_attn_seqlens_gpu import _lens
    kind, T, c = ROWS[i]
    if T.startswith("fp8"):
        import attn_fp8kv_ref as F
        import test_attn_fp8kv_gpu as FG
        t = T[len("fp8-"):]
        j = next(j for j, (t2, k2, c2) in enumerate(F.CASES) if t2 == t and c2 == c
                 and (k2 == "paged") == (kind == "paged"))
        return FG._case_call(j)[1]
    if kind == "dense":   # attn_paths row
        q, k, v = _inputs("randn", c.B, c.H, c.Hkv, c.Nq, c.Nk, c.D, None, seed=i)
        varg = v.transpose(-2, -1).contiguous() if c.vt else v
        o = torch.empty_like(q)
        return lambda: flash_attn.fmha_fwd(q, k, varg, o, v_transposed=c.vt, causal=c.causal, num_splits=c.splits)
    import test_attn_bf16_gpu as BG
    dt = torch.float16 if T == "half" else torch.bfloat16
    lens = hasattr(c, "lq")   # attn_bf16_ref.Dense rows have none
    B = len(c.lq) if lens else 2
    Nk = c.page_size * c.max_pages if kind == "paged" else c.Nk
    q, k, v = (x.to(dt) for x in _inputs("randn", B, c.H, c.Hkv, c.Nq, Nk, c.D, None, seed=i))
    kw = dict(causal=c.causal, num_splits=c.splits)
    if lens:
        kw.update(seqlens_q=_lens(c.lq), seqlens_k=_lens(c.lk))
    if kind == "paged":
        k, v, kw["block_table"] = BG.paginate(k, v, c.lk, c.page_size, c.max_pages, 0.0, seed=i)
    o = torch.empty_like(q)
    return lambda: flash_attn.fmha_fwd(q, k, v, o, **kw)


def _records(fns, trace):
    """[[(kernel name, shared memory)] of the kernels fn launches for fn in fns] from one profiler session (Kineto's
    chrome trace), split at a marker kernel launched before every call and after the last, as
    test_attn_seqlens_gpu._kernels_per_call does with the kernel names."""
    from torch.profiler import ProfilerActivity, profile
    out = []
    for _ in range(3):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            time.sleep(0.002)
            for fn in fns:
                torch.cuda._sleep(1)
                fn()
                torch.cuda.synchronize()
            torch.cuda._sleep(1)
            torch.cuda.synchronize()
            time.sleep(0.002)
        prof.export_chrome_trace(trace)
        with open(trace) as f:
            events = sorted((e for e in json.load(f)["traceEvents"] if e.get("cat") == "kernel"), key=lambda e: e["ts"])
        out = []
        for e in events:
            if e["name"] == events[0]["name"]:
                out.append([])
            else:
                out[-1].append((e["name"], e.get("args", {}).get("shared memory")))
        out = out[:-1]
        if len(out) == len(fns) and sum(e["name"] == events[0]["name"] for e in events) == len(fns) + 1:
            return out
    return out


def _profile_all_rows():
    """Child process: the kernel records of every row, as one JSON line on stdout."""
    fns = [_row_call(i) for i in range(len(ROWS))]
    with tempfile.TemporaryDirectory() as tmp:
        print("KERNEL_RECORDS " + json.dumps(_records(fns, os.path.join(tmp, "trace.json"))))


@pytest.fixture(scope="module")
def records():
    tests = Path(__file__).resolve().parent
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([str(tests.parent), str(tests)]
                                                      + [p for p in [os.environ.get("PYTHONPATH")] if p]))
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [
        "-c", "import test_attn_ring_smem_gpu as T; T._profile_all_rows()"]
    t0 = time.time()
    r = subprocess.run(cmd, cwd=tests.parent, env=env, capture_output=True, text=True, timeout=900)
    lines = [x for x in r.stdout.splitlines() if x.startswith("KERNEL_RECORDS ")]
    assert r.returncode == 0 and lines, f"profiling child failed ({r.returncode}):\n{r.stdout[-2000:]}{r.stderr[-4000:]}"
    out = json.loads(lines[-1][len("KERNEL_RECORDS "):])
    yield out
    print(f"\nshared memory of the kernel records ({len(ROWS)} rows, child {time.time() - t0:.1f} s):")
    seen = set()
    for (kind, T, c), recs in zip(ROWS, out):
        fp8 = T.startswith("fp8")
        for name, smem in recs:
            if "attn_fwd_" in name and (kind, T, c.D) not in seen:
                seen.add((kind, T, c.D))
                print(f"  {kind:<8} {T:<9} D{c.D:<5} ring {RR.ring(c.D, fp8):>2}  restated {RR.smem_bytes(c.D, fp8)}"
                      f"  record {smem}")


def test_records_carry_shared_memory(records):
    tr = [smem for recs in records for name, smem in recs if "transpose_dn_to_nd_kernel" in name]
    assert tr, "no V^T row ran the transpose pre-pass"
    assert set(tr) == {TRANSPOSE_TILE}, tr


def test_rows_cover_the_new_head_dims():
    assert {c.D for _, _, c in ROWS} == {520, 528, 776, 784, 1000, 1008}
    assert {(kind, T) for kind, T, _ in ROWS} == set(RR.KINDS)


@pytest.mark.parametrize("i", range(len(ROWS)), ids=_row_id)
def test_shared_memory_is_the_restated_one(records, i):
    kind, T, c = ROWS[i]
    fp8 = T.startswith("fp8")
    recs = records[i] if i < len(records) else []
    attn = [(name, smem) for name, smem in recs if "attn_fwd_" in name]
    assert len(attn) == 1, f"{_row_id(i)}: recorded {recs}"
    want = RR.smem_bytes(c.D, fp8)
    assert attn[0][1] == want, (f"{_row_id(i)}: the launch took {attn[0][1]} bytes of shared memory, attn_ring_ref "
                                f"restates {want} (ring {RR.ring(c.D, fp8)})")
