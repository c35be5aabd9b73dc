"""Every workload the benchmarks time, at the shape they time it, and the test that checks it there.

Sources: bench.py (the JSON line: HGEMM 8192^3, the attention rows, the host-buffer entries, the one-GPU 16384^3 point,
the next rows), leetcuda_b200.fused_ops.bench_rows (rope, rms_norm, rope of q and k, the fused RMS-norm epilogue and its
unfused pair), tools/bench_attn_causal.py, tools/bench_attn_decode.py and tools/bench_attn_seqlens.py.  SDPA / cuBLAS
columns and the multi-GPU transports are not workloads of this library's kernels and are not listed.

Shapes are read from the sources: bench.S / S16 / FA / FF, the tools' SHAPES and SWEEP (loaded with importlib; torch is
imported only inside their main).  The shapes and calls that are inline in bench_attn_causal.py, fused_ops.bench_rows
and bench.py are pinned here, together with the source text they come from (`PINNED`), which
test_bench_workload_coverage.py asserts is still there.  The seqlens tool's lengths are its own draw, reproduced.

An entry (`Workload`): id; source; row (the label the source reports it under); call (what is called, with which
shapes and arguments; `kind` selects the case of test_bench_workloads_gpu.py); check (node ids of the tests that check
the workload at that shape: `GPU_CASE` is test_bench_workloads_gpu.py::test_workload[<id>]).  `discovered()` finds the
workloads in the sources independently of the table, so that a new row, variant or shape fails the coverage gate until
it has an entry.
"""
from __future__ import annotations

import ast
import importlib.util
import re
from collections import namedtuple
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
GPU_CASE = "tests/test_bench_workloads_gpu.py::test_workload"
Workload = namedtuple("Workload", "id source row call check")


def _load(rel):
    spec = importlib.util.spec_from_file_location("bench_source_" + Path(rel).stem, ROOT / rel)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def source(rel):
    return (ROOT / rel).read_text()


BENCH = _load("bench.py")
DECODE = _load("tools/bench_attn_decode.py")
SEQLENS = _load("tools/bench_attn_seqlens.py")

BENCH_PY = "bench.py"
FUSED_PY = "leetcuda_b200/fused_ops.py"
CAUSAL_PY = "tools/bench_attn_causal.py"
DECODE_PY = "tools/bench_attn_decode.py"
SEQLENS_PY = "tools/bench_attn_seqlens.py"

# ------------------------------------------------------------------ pinned inline shapes and calls
CAUSAL_BHN = (4, 32, 4096)
CAUSAL_DS = (128, 64)
CAUSAL_DECODE = (8, 32, 8192, 128)          # Bd, Hd, Nk, D; Nq = 1
ROPE_SHAPE = (65536, 2048)
RMS_SHAPE = (131072, 2048)
FUSED_BHND = (4, 32, 4096, 128)

PINNED = {
    BENCH_PY: [
        "nsets = 2 if 8 * Bw * Hw * N * D > 200e6 else 3",
        "op(q, k, v, outs[i % nsets], 2)",
        "host_op(hq, hk, hv, ho)",
        "NSETS = 3 if world == 1 else 2",
        "op(As[j], Bs[j], Cs[j], 2, True, 2048)",
        "hgemm.hgemm_host(ha, hb, hc)",
        "op(a16[i % 2], b16[i % 2], c16, 2, True, 2048)",
    ],
    FUSED_PY: [
        "S, Hd = %d, %d" % ROPE_SHAPE,
        "R, Kk = %d, %d" % RMS_SHAPE,
        "B, H, N, D = %d, %d, %d, %d" % FUSED_BHND,
        "sets = [[t.randn(B, H, N, D, device=dev, dtype=t.half) for _ in range(3)] for _ in range(2)]",
        "attn_rmsnorm(*sets[i % 2], o, 1.0)",
        "flash_attn.fmha_fwd(*sets[i % 2], o)",
        "RN.rms_norm(o.view(-1, D), o2.view(-1, D), 1.0)",
    ],
    CAUSAL_PY: [
        "B, H, N = %d, %d, %d" % CAUSAL_BHN,
        "for D in (%d, %d):" % CAUSAL_DS,
        '"causal": lambda: flash_attn.fmha_fwd(q, k, v, o, causal=True),',
        '"full": lambda: flash_attn.fmha_fwd(q, k, v, o),',
        "Bd, Hd, Nk, D = %d, %d, %d, %d" % CAUSAL_DECODE,
        "q = torch.randn(Bd, Hd, 1, D",
        "fn = lambda: flash_attn.fmha_fwd(q, k, v, o, causal=True)",
    ],
    DECODE_PY: [
        '"auto": lambda: flash_attn.fmha_fwd(q, k, v, o, causal=causal, num_splits=0),',
        '"split1": lambda: flash_attn.fmha_fwd(q, k, v, o, causal=causal, num_splits=1),',
        '"expanded": lambda: flash_attn.fmha_fwd(q, ke, ve, o, causal=causal),',
        "if si == 0:",
        "flash_attn.fmha_fwd(q, k, v, o, causal=causal, num_splits=s)",
    ],
    SEQLENS_PY: [
        "rng = np.random.default_rng(0)",
        "lk = [int(x) for x in rng.integers(lo, hi + 1, size=B)]",
        "lq = lk if prefill else [Nq] * B",
        '"seqlens": lambda: flash_attn.fmha_fwd(q, k, v, o, causal=causal, num_splits=0, seqlens_q=tq,',
        '"padded": lambda: flash_attn.fmha_fwd(q, k, v, o, causal=causal, num_splits=0),',
        "flash_attn.fmha_fwd(qs, ks, vs, os_, causal=causal, num_splits=0)",
    ],
}


# ------------------------------------------------------------------ the library's split rule, restated
def auto_splits(B, H, Hkv, Nq, Nk, D, sms):
    """auto_splits of csrc/attn_capi.cu: split until the grid covers the SMs once, at least 4 key blocks per split, at
    most 64 splits; 1 when the grid already fills the SMs or the keys span fewer than 16 blocks."""
    ds = 64 if D <= 64 else (128 if D <= 128 else 256)
    bn, wgs = (128 if ds == 64 else 64), (1 if ds == 256 else 2)
    ctas = -(-(H // Hkv) * Nq // (64 * wgs)) * -(-D // ds) * B * Hkv
    num_kv = -(-Nk // bn)
    if ctas >= sms or num_kv < 16:
        return 1
    return max(1, min(sms // ctas, num_kv // 4, 64))


def seqlens_lengths():
    """[(lq, lk)] per SEQLENS.SHAPES entry: the tool's draw (one default_rng(0), integers(lo, hi + 1, size=B) per
    shape in order; prefill Lq = Lk, decode Lq = Nq)."""
    rng = np.random.default_rng(0)
    out = []
    for name, B, H, Hkv, Nq, Nk, D, causal, (lo, hi) in SEQLENS.SHAPES:
        lk = tuple(int(x) for x in rng.integers(lo, hi + 1, size=B))
        out.append((lk if name == "causal prefill" else (Nq,) * B, lk))
    return out


def _label(name, B, H, Hkv, Nq, Nk, D, causal):
    """The row label the tools print."""
    return f"{name} B{B} H{H} Hkv{Hkv} Nq{Nq} Nk{Nk} D{D}" + (" causal" if causal else "")


def _slug(text):
    return re.sub(r"[^A-Za-z0-9]+", "_", text).strip("_")


def _attn(op, B, H, Hkv, Nq, Nk, D, causal=False, num_splits=1, lens=None, expanded=False, sets=None):
    return {"kind": "attention", "op": op, "B": B, "H": H, "Hkv": Hkv, "Nq": Nq, "Nk": Nk, "D": D, "causal": causal,
            "num_splits": num_splits, "lens": lens, "expanded": expanded, "sets": sets}


def _bench_sets(B, H, N, D):
    return 2 if 8 * B * H * N * D > 200e6 else 3


# ------------------------------------------------------------------ the table
def _bench_entries():
    S, S16, FA, FF = BENCH.S, BENCH.S16, BENCH.FA, BENCH.FF
    FA64 = (FA[0], FA[1], FA[2], 64)
    op = BENCH.OP
    out = [
        Workload(f"hgemm_nn_{S}x{S}x{S}_fp16", BENCH_PY, "value (primary line)",
                 {"kind": "hgemm", "op": op, "M": S, "N": S, "K": S, "sets": 3, "single_out": False, "fp64": False,
                  "shards": 0},
                 ("tests/test_gemm_numerics_gpu.py::test_fp16_headline_8192", GPU_CASE)),
        Workload(f"hgemm_host_{S}x{S}x{S}_fp16", BENCH_PY, "e2e",
                 {"kind": "hgemm_host", "op": "hgemm_host", "device_op": op, "M": S, "N": S, "K": S}, (GPU_CASE,)),
        Workload(f"hgemm_nn_{S16}x{S16}x{S16}_fp16", BENCH_PY, "strong_scaling_n1",
                 {"kind": "hgemm", "op": op, "M": S16, "N": S16, "K": S16, "sets": 2, "single_out": True, "fp64": True,
                  "shards": 2},
                 (GPU_CASE,)),
        Workload("sgemm_nn_8192x8192x8192_fp32_tf32", BENCH_PY, "next_rows",
                 {"kind": "existing", "op": "sgemm_wmma_m16n16k8_mma4x2_warp2x4_stages", "M": 8192, "N": 8192,
                  "K": 8192},
                 ("tests/test_gemm_numerics_gpu.py::test_tf32_headline_8192_bench_op",)),
        Workload("merge_attn_states_T131072_H16_D128_fp16", BENCH_PY, "next_rows",
                 {"kind": "existing", "op": "merge_attn_states_cuda", "T": 131072, "H": 16, "D": 128},
                 ("tests/test_merge_numerics_gpu.py::test_bench_shape_sampled_rows",)),
    ]
    for shape, name, row, e2e in ((FA, "flash_attn_mma_stages_split_q_shared_qkv", "secondary", True),
                                  (FF, "ffpa_mma_acc_f32_L1", "config4", True),
                                  (FA64, "flash_attn_mma_stages_split_q_shared_qkv", "secondary_d64", False)):
        B, H, N, D = shape
        out.append(Workload(f"attn_fwd_B{B}_H{H}_N{N}_D{D}_fp16", BENCH_PY, row,
                            _attn(name, B, H, H, N, N, D, sets=_bench_sets(B, H, N, D)), (GPU_CASE,)))
        if e2e:
            out.append(Workload(f"fmha_host_B{B}_H{H}_N{N}_D{D}_fp16", BENCH_PY, row + ".e2e",
                                {"kind": "fmha_host", "op": "fmha_host", "device_op": name, "B": B, "H": H, "N": N,
                                 "D": D},
                                (GPU_CASE,)))
    Sr, Hd = ROPE_SHAPE
    R, K = RMS_SHAPE
    B, H, N, D = FUSED_BHND
    out += [
        Workload(f"rope_seq{Sr}_hidden{Hd}_fp32", FUSED_PY, "next_rows",
                 {"kind": "existing", "op": "rope_f32x4_pack", "S": Sr, "hidden": Hd},
                 ("tests/test_rope_rms_numerics_gpu.py::test_rope_f32_bench_shape_sampled_rows",)),
        Workload(f"rms_norm_rows{R}_K{K}_fp16", FUSED_PY, "next_rows",
                 {"kind": "existing", "op": "rms_norm_f16x8_pack_f32", "rows": R, "K": K},
                 ("tests/test_rope_rms_numerics_gpu.py::test_rms_norm_bench_shape_sampled_rows",)),
        Workload(f"rope_qk_B{B}_H{H}_N{N}_D{D}_fp16", FUSED_PY, "next_rows",
                 {"kind": "existing", "op": "rope_qk", "B": B, "H": H, "N": N, "D": D},
                 ("tests/test_rope_rms_numerics_gpu.py::test_rope_qk_bench_shape_sampled_heads",)),
        Workload(f"attn_rmsnorm_B{B}_H{H}_N{N}_D{D}_fp16", FUSED_PY, "next_rows",
                 {"kind": "rms", "op": "attn_rmsnorm", "B": B, "H": H, "N": N, "D": D, "g": 1.0, "sets": 2},
                 (GPU_CASE,)),
        Workload(f"attn_rmsnorm_B{B}_H{H}_N{N}_D{D}_fp16:unfused", FUSED_PY, "next_rows (unfused)",
                 {"kind": "rms", "op": "fmha_fwd+rms_norm", "B": B, "H": H, "N": N, "D": D, "g": 1.0, "sets": 2},
                 (GPU_CASE,)),
    ]
    return out


def _causal_entries():
    B, H, N = CAUSAL_BHN
    out = []
    for D in CAUSAL_DS:
        for variant, causal in (("causal", True), ("full", False)):
            out.append(Workload(f"causal_tool/B{B}_H{H}_N{N}_D{D}/{variant}", CAUSAL_PY, f"B{B} H{H} N{N} D{D}: {variant}",
                                _attn("fmha_fwd", B, H, H, N, N, D, causal=causal), (GPU_CASE,)))
    Bd, Hd, Nk, D = CAUSAL_DECODE
    out.append(Workload(f"causal_tool/decode_B{Bd}_H{Hd}_Nq1_Nk{Nk}_D{D}", CAUSAL_PY,
                        f"decode B{Bd} H{Hd} Nq1 Nk{Nk} D{D}", _attn("fmha_fwd", Bd, Hd, Hd, 1, Nk, D, causal=True),
                        (GPU_CASE,)))
    return out


DECODE_VARIANTS = {"auto": dict(num_splits=0), "split1": dict(num_splits=1), "expanded": dict(expanded=True)}
SEQLENS_VARIANTS = ("seqlens", "padded", "loop")


def _decode_entries():
    out = []
    for si, (name, B, H, Hkv, Nq, Nk, D, causal) in enumerate(DECODE.SHAPES):
        label = _label(name, B, H, Hkv, Nq, Nk, D, causal)
        variants = dict(DECODE_VARIANTS)
        if si == 0:
            variants.update({f"splits{s}": dict(num_splits=s) for s in DECODE.SWEEP})
        for variant, kw in variants.items():
            out.append(Workload(f"decode_tool/{_slug(label)}/{variant}", DECODE_PY, f"{label}: {variant}",
                                _attn("fmha_fwd", B, H, Hkv, Nq, Nk, D, causal=causal, **kw), (GPU_CASE,)))
    return out


def _seqlens_entries():
    out = []
    for (name, B, H, Hkv, Nq, Nk, D, causal, _), lens in zip(SEQLENS.SHAPES, seqlens_lengths()):
        label = _label(name, B, H, Hkv, Nq, Nk, D, causal)
        for variant in SEQLENS_VARIANTS:
            op = "fmha_fwd_loop" if variant == "loop" else "fmha_fwd"
            out.append(Workload(f"seqlens_tool/{_slug(label)}/{variant}", SEQLENS_PY, f"{label}: {variant}",
                                _attn(op, B, H, Hkv, Nq, Nk, D, causal=causal, num_splits=0,
                                      lens=None if variant == "padded" else lens),
                                (GPU_CASE,)))
    return out


WORKLOADS = _bench_entries() + _causal_entries() + _decode_entries() + _seqlens_entries()
BY_ID = {w.id: w for w in WORKLOADS}


# ------------------------------------------------------------------ the workloads the sources run
def _runs_keys(text):
    """Keys of a tool's `runs` dict whose callable is this library's (the SDPA columns excluded)."""
    keys = []
    for m in re.finditer(r'^\s+"(\w+)": (lambda\b.*|loop,)$', text, re.M):
        if "scaled_dot_product_attention" not in m.group(2):
            keys.append(m.group(1))
    return keys


def _bench_discovered():
    """id -> op name of bench.py's and fused_ops.bench_rows' rows, found by walking their syntax trees: every
    attention_row call (its shape evaluated in bench.py's namespace, its e2e flag), every constant `workload` of a row
    config (the multi-GPU line's is a format string and is out of scope), a row with an `unfused` pair, the host GEMM."""
    found = {}
    ns = vars(BENCH)
    for rel in (BENCH_PY, FUSED_PY):
        tree = ast.parse(source(rel))
        for node in ast.walk(tree):
            if isinstance(node, ast.Call) and isinstance(node.func, ast.Name) and node.func.id == "attention_row":
                B, H, N, D = eval(compile(ast.Expression(node.args[6]), rel, "eval"), ns)
                found[f"attn_fwd_B{B}_H{H}_N{N}_D{D}_fp16"] = node.args[8].value
                if node.args[15].value:
                    found[f"fmha_host_B{B}_H{H}_N{N}_D{D}_fp16"] = "fmha_host"
            elif isinstance(node, ast.Call) and isinstance(node.func, ast.Attribute) and node.func.attr == "hgemm_host":
                found[f"hgemm_host_{BENCH.S}x{BENCH.S}x{BENCH.S}_fp16"] = "hgemm_host"
            elif isinstance(node, ast.Dict):
                keys = [k.value for k in node.keys if isinstance(k, ast.Constant)]
                if "workload" in keys:
                    val = node.values[keys.index("workload")]
                    if isinstance(val, ast.Constant):
                        opv = node.values[keys.index("op")] if "op" in keys else None
                        found[val.value.split(" ")[0]] = opv.value if isinstance(opv, ast.Constant) else None
                if "unfused" in keys:
                    inner = [n for n in ast.walk(node) if isinstance(n, ast.Dict) and n is not node]
                    for d in inner:
                        ks = [k.value for k in d.keys if isinstance(k, ast.Constant)]
                        if "workload" in ks and isinstance(d.values[ks.index("workload")], ast.Constant):
                            found[d.values[ks.index("workload")].value + ":unfused"] = "fmha_fwd+rms_norm"
    return found


def discovered():
    """{id: op or None} of every workload the bench sources time, found without the table."""
    found = _bench_discovered()
    text = source(CAUSAL_PY)
    B, H, N = (int(x) for x in re.search(r"B, H, N = (\d+), (\d+), (\d+)", text).groups())
    Ds = [int(x) for x in re.search(r"for D in \(([\d, ]+)\):", text).group(1).split(",") if x.strip()]
    for D in Ds:
        for variant in _runs_keys(text):
            found[f"causal_tool/B{B}_H{H}_N{N}_D{D}/{variant}"] = "fmha_fwd"
    m = re.search(r"Bd, Hd, Nk, D = (\d+), (\d+), (\d+), (\d+)", text)
    if m:
        Bd, Hd, Nk, D = (int(x) for x in m.groups())
        found[f"causal_tool/decode_B{Bd}_H{Hd}_Nq1_Nk{Nk}_D{D}"] = "fmha_fwd"
    text = source(DECODE_PY)
    variants = _runs_keys(text)
    for si, (name, Bb, Hh, Hkv, Nq, Nk, D, causal) in enumerate(DECODE.SHAPES):
        vs = variants + ([f"splits{s}" for s in DECODE.SWEEP] if si == 0 and "if si == 0:" in text else [])
        for variant in vs:
            found[f"decode_tool/{_slug(_label(name, Bb, Hh, Hkv, Nq, Nk, D, causal))}/{variant}"] = "fmha_fwd"
    text = source(SEQLENS_PY)
    variants = _runs_keys(text)
    for name, Bb, Hh, Hkv, Nq, Nk, D, causal, _ in SEQLENS.SHAPES:
        for variant in variants:
            found[f"seqlens_tool/{_slug(_label(name, Bb, Hh, Hkv, Nq, Nk, D, causal))}/{variant}"] = \
                "fmha_fwd_loop" if variant == "loop" else "fmha_fwd"
    return found
