"""The GEMM kernel in two-CTA clusters (csrc/hgemm_sm90.cuh): the two CTAs of a cluster take the two m-tiles of a pair
tile, and each multicasts half of the shared B tile into both CTAs' shared memory.  Checked against the fp64 reference
of gemm_ref.py (bit for bit for the probes), with guard bands around C, on:

  * cluster size 1 (a single m-tile) and 2, every instantiation under clusters of two;
  * a lone partner: an odd tiles_m puts the last cluster's second m-tile past M (zero A boxes, no stores), in NN, TN and
    TF32;
  * several cluster tiles per cluster, and single-k-block tiles with more tiles per cluster than the ring has stages,
    so that remote releases of a stage cross tile boundaries;
  * N tails inside the multicast halves of B: the first half partial (the second one entirely past N), and the second
    half partial;
  * the same bits from a cluster of one as from a cluster of two, and the peer-store epilogue of the fused all-gather
    under clusters with a lone partner.

test_shape_table_coverage restates the host's choice of cluster size, tile width and grid (hgemm_capi.cu) and checks
that the table reaches each of these cases on 132 SMs.
"""
import ctypes

import numpy as np
import pytest
import torch

import gemm_ref as R
from leetcuda_b200 import _capi, hgemm, sgemm

MARGIN = 256
SENT16, SENT32 = 0x7E5B, 0x7FA5A5A5
# (mode, B given as [N,K] storage); TF32 B is [N,K] in the kernel either way
CALLS = [("f16", False), ("f16", True), ("f16acc", False), ("f16acc", True), ("tf32", True)]
# M x N x K.  On 132 SMs (see test_shape_table_coverage; clusters of two at most 66 at once):
#   100 x 520 x 136     one m-tile: cluster size 1
#   2600 x 2344 x 136   21 m-tiles (lone partner), 256-column tile, 2 cluster tiles per cluster, N tail 40: first half
#                       of the last B tile partial, second half past N
#   2600 x 2440 x 72    the same with N tail 136: second half partial
#   2600 x 2000 x 136   128-column tile, lone partner, 3 cluster tiles per cluster, N tail 80 (second 64-row half)
#   8192 x 4096 x 8     256-column tile, one k-block per tile, 8 cluster tiles per cluster through the 4-stage ring
#   8576 x 1416 x 8     128-column tile, one k-block, 7 cluster tiles per cluster through the 6-stage ring, 67 m-tiles
#   300 x 264 x 200     3 m-tiles: one full pair and a lone partner, one tile per cluster
SHAPES = [(100, 520, 136), (2600, 2344, 136), (2600, 2440, 72), (2600, 2000, 136), (8192, 4096, 8), (8576, 1416, 8),
          (300, 264, 200)]
GENS = ("randn", "k_probe", "a_probe")


def plan(M, N, sms, max_clusters):
    """The host's launch for an M x N output, restated (hgemm_impl and launch_hgemm): cluster size cs = 2 when there
    are two m-tiles to pair; 128 x 256 tiles unless 0.9 x the last-wave occupancy of 128 x 128 tiles beats it, where a
    lone partner's padded m-tile counts as launched but not as work; a persistent grid of min(cluster tiles, #SMs) CTAs
    (cs = 1) or min(cluster tiles, max_clusters) clusters (cs = 2)."""
    tm = -(-M // R.BM)
    cs = 2 if tm >= 2 else 1

    def score(bn, eff):
        tn = -(-N // bn)
        waves = -(-(-(-tm // cs) * cs * tn) // sms)
        return eff * tm * tn / (waves * sms)
    bn = 128 if score(128, 0.90) > score(256, 1.0) else 256
    tn = -(-N // bn)
    tiles = -(-tm // cs) * tn
    clusters = min(tiles, sms if cs == 1 else max_clusters)
    return {"cs": cs, "bn": bn, "tiles_m": tm, "tiles_n": tn, "cluster_tiles": tiles, "grid": cs * clusters,
            "per_cluster": -(-tiles // clusters), "lone": cs == 2 and tm % 2 == 1, "n_tail": N % bn}


def test_shape_table_coverage():
    """On 132 SMs, with at most 66 clusters of two at once (fewer only adds cluster tiles per cluster), the table
    reaches: cluster size 1 in NN, TN and TF32; every instantiation in clusters of two with several cluster tiles per
    cluster and with single-k-block tiles wrapping the ring; a lone partner in NN, TN and TF32 at both tile widths;
    N tails in the first and in the second half of B at both tile widths."""
    sms, slots = 132, 66
    single, paired, multi, wrapped, lone, tails = set(), set(), set(), set(), set(), set()
    for M, N, K in SHAPES:
        p = plan(M, N, sms, slots)
        for mode, tn in CALLS:
            inst = R.instantiation(mode, tn, p["bn"])
            layout = "tf32" if mode == "tf32" else ("TN" if tn else "NN")
            if p["cs"] == 1:
                single.add(layout)
                continue
            paired.add(inst)
            if p["per_cluster"] > 1:
                multi.add(inst)
            if -(-K // R.KBLOCK[mode]) == 1 and p["per_cluster"] > R.STAGES[p["bn"]]:
                wrapped.add(inst)
            if p["lone"]:
                lone.add((layout, p["bn"]))
            if p["n_tail"]:
                tails.add((p["bn"], "first" if p["n_tail"] < p["bn"] // 2 else "second"))
    assert single == {"NN", "TN", "tf32"}
    assert paired == multi == wrapped == R.ALL_INSTANTIATIONS
    assert lone == {(lay, bn) for lay in ("NN", "TN", "tf32") for bn in (128, 256)}
    assert tails == {(bn, h) for bn in (128, 256) for h in ("first", "second")}


# ------------------------------------------------------------------ GPU
def _guarded(shape, dtype):
    n = int(np.prod(shape))
    buf = torch.empty(n + 2 * MARGIN, dtype=dtype, device="cuda")
    buf.view(torch.int16 if dtype == torch.float16 else torch.int32).fill_(SENT16 if dtype == torch.float16 else SENT32)
    return buf, buf[MARGIN:MARGIN + n].view(shape)


def _untouched(t):
    if t.dtype == torch.float16:
        return bool((t.view(torch.int16) == SENT16).all())
    return bool((t.view(torch.int32) == SENT32).all())


def _call(mode, tn, a, b, c):
    K, N = b.shape
    if mode == "tf32":
        sgemm.sgemm_tf32(a.clone(), b.t().contiguous().view(K, N), c, tn=True, round_inputs=True)
    else:
        hgemm.hgemm(a, b.t().reshape(K, N).contiguous() if tn else b, c, tn=tn,
                    acc="f16" if mode == "f16acc" else "f32")


@pytest.mark.gpu
@pytest.mark.parametrize("gen", GENS)
@pytest.mark.parametrize("shape", SHAPES, ids=[f"{m}x{n}x{k}" for m, n, k in SHAPES])
def test_clusters(shape, gen):
    M, N, K = shape
    inputs = {}
    for mode, tn in CALLS:
        dt = np.float32 if mode == "tf32" else np.float16
        if dt not in inputs:
            a_np, b_np, info = R.make_inputs(gen, M, N, K, dt, seed=M + 7 * N + 31 * K + 1000 * GENS.index(gen))
            inputs[dt] = (torch.from_numpy(a_np).cuda(), torch.from_numpy(b_np).cuda(), info)
        a, b, info = inputs[dt]
        buf, c = _guarded((M, N), torch.float32 if mode == "tf32" else torch.float16)
        _call(mode, tn, a, b, c)
        torch.cuda.synchronize()
        what = f"{M}x{N}x{K} {gen} {mode} {'TN' if tn else 'NN'}"
        assert _untouched(buf[:MARGIN]) and _untouched(buf[-MARGIN:]), f"{what}: store outside C"
        ref = R.reference(a, b, mode)
        if gen in R.EXACT:
            if not torch.equal(c.double(), ref["c"]):
                pytest.fail(f"{what}: " + R.probe_miss(a.cpu().numpy(), b.cpu().numpy(), c.cpu().double().numpy(),
                                                        ref["c"].cpu().numpy(), info))
            continue
        err = (c.double() - ref["c"]).abs()
        bound = R.bound(ref)
        if not bool((err <= bound).all()):
            r = torch.nan_to_num(err / bound, nan=float("inf"))
            at = np.unravel_index(int(r.argmax()), tuple(r.shape))
            pytest.fail(f"{what}: |err|/bound {r.max().item():.3g} at {at}")


@pytest.mark.gpu
@pytest.mark.parametrize("tn", [False, True])
def test_cluster_sizes_agree(tn):
    """Row shards of one m-tile run in clusters of one; the full product runs in clusters of two, with a lone partner
    (9 m-tiles).  Their rows of C are the same bits."""
    M, N, K = 1100, 776, 520
    a_np, b_np, _ = R.make_inputs("randn", M, N, K, np.float16, seed=5)
    a, b = torch.from_numpy(a_np).cuda(), torch.from_numpy(b_np).cuda()
    barg = b.t().reshape(K, N).contiguous() if tn else b
    full = torch.empty(M, N, dtype=torch.half, device="cuda")
    hgemm.hgemm(a, barg, full, tn=tn)
    layout = _capi.B_ROW_MAJOR_NK if tn else _capi.B_ROW_MAJOR_KN
    for row0, rows in ((0, 128), (384, 100), (1024, 76)):
        buf, c = _guarded((M, N), torch.half)
        rc = _capi.lib().b200_hgemm_f16_rows(a[row0:row0 + rows].data_ptr(), barg.data_ptr(), c.data_ptr(), rows, N,
                                             K, layout, row0, torch.cuda.current_stream().cuda_stream)
        assert rc == 0, _capi.last_error()
        torch.cuda.synchronize()
        assert torch.equal(c[row0:row0 + rows].view(torch.int16), full[row0:row0 + rows].view(torch.int16))
        assert _untouched(buf[:MARGIN + row0 * N]) and _untouched(buf[MARGIN + (row0 + rows) * N:])


@pytest.mark.gpu
@pytest.mark.parametrize("tn", [False, True])
def test_fused_epilogue_lone_partner(tn):
    """The peer-store epilogue of b200_hgemm_f16_rows_fused with a 300-row shard (3 m-tiles: a pair and a lone
    partner): C and both stand-in peer buffers get the shard rows bit for bit, within the bound, and nothing else."""
    rows, N, K, row0, mtot = 300, 264, 136, 50, 400
    a_np, b_np, _ = R.make_inputs("randn", rows, N, K, np.float16, seed=87)
    a, b = torch.from_numpy(a_np).cuda(), torch.from_numpy(b_np).cuda()
    barg = b.t().reshape(K, N).contiguous() if tn else b
    bufs = [_guarded((mtot, N), torch.half) for _ in range(3)]
    peers = (ctypes.c_void_p * 2)(*[v.data_ptr() for _, v in bufs[1:]])
    rc = _capi.lib().b200_hgemm_f16_rows_fused(
        a.data_ptr(), barg.data_ptr(), bufs[0][1].data_ptr(), None, peers, 2, rows, N, K,
        _capi.B_ROW_MAJOR_NK if tn else _capi.B_ROW_MAJOR_KN, row0, torch.cuda.current_stream().cuda_stream)
    assert rc == 0, _capi.last_error()
    torch.cuda.synchronize()
    shard = bufs[0][1][row0:row0 + rows]
    ref = R.reference(a, b, "f16")
    assert bool(((shard.double() - ref["c"]).abs() <= R.bound(ref)).all())
    for i, (buf, view) in enumerate(bufs):
        assert torch.equal(view[row0:row0 + rows].view(torch.int16), shard.view(torch.int16)), f"buffer {i}"
        assert _untouched(buf[:MARGIN + row0 * N]) and _untouched(buf[MARGIN + (row0 + rows) * N:]), f"buffer {i}"
