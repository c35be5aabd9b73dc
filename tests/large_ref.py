"""The large-tensor case table: every entry family run where an element offset passes 2^31 or a byte offset passes 2^32,
and at the grid limits (B * Hkv = 65535).

Each case restates, from its shapes alone, the device bytes the GPU test allocates (`peak`: the tensors the test holds
while the call runs, NaN guard bands included, and `scratch`: the stream-ordered scratch the library allocates inside
the call, which torch's allocator does not see) and, per buffer the checked region reads or writes, the largest
element offset there (`offsets`: (buffer, element offset, bytes per element)), from the layout:

    dense / seqlens / rms   Q, O [B, H, N, D]           (b*H + h)*N*D + t*D + d;  K, V [B, Hkv, Nk, D] likewise
    split workspace         ws_o [S, B*H*Nq, D] fp32     (s*B*H*Nq + (b*H + h)*Nq + t)*D + d
    paged pool              [P, page_size, Hkv, D]       (page*page_size + r)*Hkv*D + h*D + d
    varlen                  q, o [total_q, H, D]         (row*H + h)*D + d;  k, v [total_k, Hkv, D]
    gemm C                  [M, N]                       row*N + col  (_rows: (row0 + r)*N + col)
    merge                   [T, H, D]                    (t*H + h)*D + d
    rope / rms_norm / round [rows, D]                    row*D + d

The checked regions always include the last row, head or page of the buffer, so the largest offset is the last
element of the buffer (numel - 1) unless the case says otherwise.  test_large_coverage.py checks the table on the CPU;
test_large_gpu.py runs it on the GPU.  Nothing here imports torch.cuda.
"""
from __future__ import annotations

from dataclasses import dataclass, field

GiB = 2 ** 30
PEAK_LIMIT = 20 * GiB
TWO31 = 2 ** 31
TWO32 = 2 ** 32
GUARD = 4096                         # NaN guard elements after every output
ELEM = {"f16": 2, "bf16": 2, "f32": 4, "e4m3": 1, "i32": 4}

FAMILIES = {
    "dense": "fmha_fwd fp16 / bf16, grouped-query, causal with lse; split-KV with a > 4 GiB fp32 workspace",
    "seqlens": "fmha_fwd(seqlens_q=, seqlens_k=) over a padded KV cache, decoding",
    "long_context": "one sequence, Hkv 1, D 128, Nk = 2^24 + 77, with and without splits",
    "paged": "fmha_fwd(block_table=) fp16 / bf16 over a > 2^31-element pool",
    "fp8": "fmha_fwd with float8_e4m3fn K/V of > 2^32 bytes: a paged pool and a padded per-sequence cache",
    "varlen": "fmha_varlen_fwd with total_q*H*D and total_k*Hkv*D > 2^31, and over a paged pool of > 2^31 elements",
    "rms_attn": "attn_rmsnorm with O > 2^31 elements",
    "grid_edge": "B*Hkv = 65535 exactly: dense, seqlens, paged and varlen",
    "hgemm": "hgemm f16, f16acc and _rows with C > 2^31 elements",
    "sgemm": "sgemm_tf32 NN / TN and 3xtf32 with C > 2^31 elements, and K past the TF32 transpose's old grid limit",
    "elementwise": "merge_attn_states (f16, bf16, f32), rope_f32, rope_qk, rms_norm (f16, f32), tf32_round",
}

# The entry points each family must reach (family -> entries; a case names one).
ENTRIES = {
    "dense": {"fmha_f16_gqa", "fmha_bf16", "fmha_f16_split"},
    "seqlens": {"fmha_f16_seqlens"},
    "long_context": {"fmha_f16_gqa_long"},
    "paged": {"fmha_f16_paged", "fmha_bf16_paged"},
    "fp8": {"fmha_f16_fp8kv_paged", "fmha_f16_fp8kv_seqlens"},
    "varlen": {"fmha_f16_varlen", "fmha_f16_varlen_paged"},
    "rms_attn": {"attn_rmsnorm"},
    "grid_edge": {"fmha_f16_edge", "fmha_bf16_seqlens_edge", "fmha_f16_paged_edge", "fmha_f16_varlen_edge"},
    "hgemm": {"hgemm_f16", "hgemm_f16acc", "hgemm_f16_rows"},
    "sgemm": {"sgemm_tf32_nn", "sgemm_tf32_tn", "sgemm_3xtf32", "sgemm_tf32_nn_longk", "sgemm_tf32_nn_noround_longk",
              "sgemm_3xtf32_longk", "sgemm_tf32_nn_kedge"},
    "elementwise": {"merge_f16", "merge_bf16", "merge_f32", "rope_f32", "rope_qk", "rms_norm_f16", "rms_norm_f32",
                    "tf32_round"},
}


@dataclass(frozen=True)
class Case:
    name: str
    family: str
    entry: str
    dtype: str
    shape: dict
    peak: int                        # bytes of torch tensors held during the call
    offsets: tuple                   # ((buffer, largest element offset of the checked region, bytes per element), ...)
    past: bool                       # the checked region passes 2^31 elements and 2^32 bytes in some buffer
    scratch: int = 0                 # bytes the library allocates inside the call
    note: str = ""
    extra: dict = field(default_factory=dict)

    @property
    def total(self):
        return self.peak + self.scratch


def out_bytes(numel, dtype):
    """An output with its guard band."""
    return (numel + GUARD) * ELEM[dtype]


def last(numel):
    return numel - 1


# ------------------------------------------------------------------ attention
def _dense(name, entry, dtype, B, H, Hkv, N, D, causal=True, splits=1):
    q = B * H * N * D
    kv = B * Hkv * N * D
    e = ELEM[dtype]
    lse = B * H * N
    peak = q * e + out_bytes(q, dtype) + 2 * kv * e + out_bytes(lse, "f32")
    scratch = splits * (q + lse) * 4 if splits > 1 else 0
    offs = [("q", last(q), e), ("o", last(q), e), ("k", last(kv), e)]
    if splits > 1:
        offs.append(("ws_o", last(splits * q), 4))
    return Case(name, "dense", entry, dtype, dict(B=B, H=H, Hkv=Hkv, Nq=N, Nk=N, D=D, causal=causal, splits=splits),
                peak, tuple(offs), past=q >= TWO31, scratch=scratch)


def _seqlens_lengths(B, Nq, Nk):
    """Ragged decode lengths, the longest sequence last."""
    lq = [1 + (b * 5) % Nq for b in range(B)]
    lk = [1 + (b * 7919) % (Nk - 1) for b in range(B)]
    lq[-1], lk[-1] = Nq, Nk
    lk[0] = 0
    return lq, lk


def _seqlens(name, family, entry, B, H, Hkv, Nq, Nk, D, dtype="f16", kvdtype="f16", scales=(1.0, 1.0)):
    q, kv, e, ekv = B * H * Nq * D, B * Hkv * Nk * D, ELEM[dtype], ELEM[kvdtype]
    lse = B * H * Nq
    peak = q * e + out_bytes(q, dtype) + 2 * kv * ekv + out_bytes(lse, "f32") + 2 * B * 4
    lq, lk = _seqlens_lengths(B, Nq, Nk)
    return Case(name, family, entry, dtype,
                dict(B=B, H=H, Hkv=Hkv, Nq=Nq, Nk=Nk, D=D, causal=True, splits=1, lq=lq, lk=lk, kv=kvdtype,
                     k_scale=scales[0], v_scale=scales[1]), peak,
                (("k", last(kv), ekv), ("v", last(kv), ekv)), past=kv >= TWO31 and kv * ekv >= TWO32)


def _long(name, Nk, H=8, D=128, splits=(1, 64)):
    kv = Nk * D
    q = H * D
    peak = 2 * kv * 2 + q * 2 + len(splits) * (out_bytes(q, "f16") + out_bytes(H, "f32"))
    scratch = max(splits) * (q + H) * 4
    tail = -(-TWO31 // D)                 # the first key row at or past 2^31 elements
    return Case(name, "long_context", "fmha_f16_gqa_long", "f16",
                dict(B=1, H=H, Hkv=1, Nq=1, Nk=Nk, D=D, causal=False, splits=splits, tail=tail), peak,
                (("k", last(kv), 2), ("v", last(kv), 2)), past=kv >= TWO31, scratch=scratch,
                note="the keys from row `tail` on (past 2^31 elements) carry all but ~e^-90 of every query's softmax "
                     "weight, so a misread of any of them moves O by O(|V|)")


def _paged(name, family, entry, qdtype, kvdtype, num_pages, page_size, Hkv, D, B, H, Nq, max_pages, scales=(1.0, 1.0)):
    pool = num_pages * page_size * Hkv * D
    q = B * H * Nq * D
    lse = B * H * Nq
    eq, ekv = ELEM[qdtype], ELEM[kvdtype]
    peak = 2 * pool * ekv + q * eq + out_bytes(q, qdtype) + out_bytes(lse, "f32") + B * max_pages * 4 + 2 * B * 4
    lq, lk = _seqlens_lengths(B, Nq, max_pages * page_size)
    return Case(name, family, entry, qdtype,
                dict(B=B, H=H, Hkv=Hkv, Nq=Nq, D=D, num_pages=num_pages, page_size=page_size, max_pages=max_pages,
                     kv=kvdtype, causal=True, lq=lq, lk=lk, k_scale=scales[0], v_scale=scales[1]), peak,
                (("k_pool", last(pool), ekv), ("v_pool", last(pool), ekv)), past=pool >= TWO31 and pool * ekv >= TWO32,
                note="the block tables take the top pages of the pool, the last sequence its very last page")


def _varlen_lengths(B, base):
    lens = [base + (b * 37) % 64 - 32 for b in range(B)]
    lens[-1] = base + 76
    return lens


def _varlen(name, B, H, Hkv, D, base):
    lens = _varlen_lengths(B, base)
    total = sum(lens)
    q, kv = total * H * D, total * Hkv * D
    lse = H * total
    peak = q * 2 + out_bytes(q, "f16") + 2 * kv * 2 + out_bytes(lse, "f32") + 2 * (B + 1) * 4
    return Case(name, "varlen", "fmha_f16_varlen", "f16", dict(B=B, H=H, Hkv=Hkv, D=D, lens=lens, causal=True), peak,
                (("q", last(q), 2), ("o", last(q), 2), ("k", last(kv), 2)), past=min(q, kv) >= TWO31)


def _varlen_paged(name, num_pages, page_size, Hkv, D, H, lq, max_pages):
    pool = num_pages * page_size * Hkv * D
    B, total = len(lq), sum(lq)
    q, lse = total * H * D, H * total
    peak = 2 * pool * 2 + q * 2 + out_bytes(q, "f16") + out_bytes(lse, "f32") + B * max_pages * 4 + (2 * B + 1) * 4
    lk = [max_pages * page_size - 1 - 97 * b for b in range(B)]
    lk[-1] = max_pages * page_size
    return Case(name, "varlen", "fmha_f16_varlen_paged", "f16",
                dict(B=B, H=H, Hkv=Hkv, D=D, num_pages=num_pages, page_size=page_size, max_pages=max_pages, lq=lq,
                     lk=lk, causal=True), peak,
                (("k_pool", last(pool), 2), ("v_pool", last(pool), 2)), past=pool >= TWO31,
                note="the block tables take the top pages of the pool, the last sequence its very last page")


def _rms(name, B, H, N, D):
    q = B * H * N * D
    peak = 3 * q * 2 + out_bytes(q, "f16")
    return Case(name, "rms_attn", "attn_rmsnorm", "f16", dict(B=B, H=H, Hkv=H, Nq=N, Nk=N, D=D, g=1.5), peak,
                (("o", last(q), 2),), past=q >= TWO31)


def _edge(name, entry, dtype, B, H, Hkv, N, D, kind):
    q, kv = B * H * N * D, B * Hkv * N * D
    lse = B * H * N
    peak = q * 2 + out_bytes(q, dtype) + 2 * kv * 2 + out_bytes(lse, "f32") + (B + 1) * 4 * 2 + B * 4
    return Case(name, "grid_edge", entry, dtype, dict(B=B, H=H, Hkv=Hkv, Nq=N, Nk=N, D=D, kind=kind), peak,
                (("o", last(q), 2),), past=False, note="B * Hkv = 65535, the largest grid.y")


# ------------------------------------------------------------------ GEMM
def _hgemm(name, entry, M, N, K, rows=None, acc="f32", tn=False):
    c = M * N
    arows = rows if rows else M
    peak = arows * K * 2 + K * N * 2 + out_bytes(c, "f16")
    row0 = M - rows if rows else 0
    return Case(name, "hgemm", entry, "f16", dict(M=M, N=N, K=K, rows=rows, row0=row0, acc=acc, tn=tn), peak,
                (("c", last(c), 2),), past=c >= TWO31, note="_rows: row0 * N > 2^31" if rows else "")


def _sgemm(name, entry, M, N, K, mode, tn=False, rnd=True, gen="randn"):
    c = M * N
    peak = M * K * 4 + K * N * 4 + out_bytes(c, "f32")
    if mode == "3xtf32":
        scratch = (M * 3 * K + 3 * K * N) * 4
    else:
        scratch = 0 if tn else K * N * 4
    offs = [("c", last(c), 4), ("b", last(K * N), 4), ("bt", last(3 * K * N if mode == "3xtf32" else K * N), 4)]
    return Case(name, "sgemm", entry, "f32", dict(M=M, N=N, K=K, mode=mode, tn=tn, round=rnd, gen=gen), peak,
                tuple(offs), past=c >= TWO31, scratch=scratch)


# ------------------------------------------------------------------ elementwise
def _merge(name, dtype, T, H, D, in_place):
    n, e = T * H * D, ELEM[dtype]
    lse = H * T
    peak = (1 if in_place else 2) * n * e + out_bytes(n, dtype) + 2 * lse * 4 + out_bytes(lse, "f32")
    return Case(name, "elementwise", f"merge_{dtype}", dtype, dict(T=T, H=H, D=D, in_place=in_place), peak,
                (("o", last(n), e),), past=n >= TWO31, note="output is prefix_output" if in_place else "")


def _rows(name, entry, dtype, rows, D, in_place, extra=None):
    n, e = rows * D, ELEM[dtype]
    peak = out_bytes(n, dtype) + (0 if in_place else n * e)
    return Case(name, "elementwise", entry, dtype, dict(rows=rows, D=D, in_place=in_place, **(extra or {})), peak,
                (("x", last(n), e),), past=n >= TWO31)


def _rope_qk(name, B, H, N, D):
    n = B * H * N * D
    peak = 2 * out_bytes(n, "f16")
    return Case(name, "elementwise", "rope_qk", "f16", dict(B=B, H=H, N=N, D=D), peak,
                (("q", last(n), 2), ("k", last(n), 2)), past=n >= TWO31, note="in place")


_SPLIT_N = (2 ** 29 + 2 ** 20) // (64 * 8 * 128)        # Q of 2^29 + 2^20 elements: an fp32 workspace of > 4 GiB

CASES = [
    _dense("dense_f16_gqa_causal", "fmha_f16_gqa", "f16", 512, 16, 2, 1040, 256),
    _dense("dense_bf16_gqa_causal", "fmha_bf16", "bf16", 512, 16, 2, 1040, 256),
    _dense("dense_f16_split2", "fmha_f16_split", "f16", 64, 8, 2, _SPLIT_N, 128, causal=False, splits=2),
    _seqlens("seqlens_f16_decode", "seqlens", "fmha_f16_seqlens", 64, 32, 8, 4, 33000, 128),
    _long("long_context_f16", 2 ** 24 + 77),
    _paged("paged_f16", "paged", "fmha_f16_paged", "f16", "f16", 131073, 16, 8, 128, 4, 32, 2, 64),
    _paged("paged_bf16", "paged", "fmha_bf16_paged", "bf16", "bf16", 131073, 16, 8, 128, 4, 32, 2, 64),
    _paged("fp8_paged_f16", "fp8", "fmha_f16_fp8kv_paged", "f16", "e4m3", 262145, 16, 8, 128, 4, 32, 2, 64,
           scales=(0.37, 1.75)),
    _seqlens("fp8_seqlens_f16", "fp8", "fmha_f16_fp8kv_seqlens", 64, 16, 8, 4, 65600, 128, kvdtype="e4m3",
             scales=(0.37, 1.75)),
    _varlen("varlen_f16_causal", 1025, 16, 16, 128, 1024),
    _varlen_paged("varlen_paged_f16", 131073, 16, 8, 128, 32, [5, 17, 1, 64], 64),
    _rms("rms_attn_f16", 512, 16, 1040, 256),
    _edge("edge_dense_f16", "fmha_f16_edge", "f16", 65535, 1, 1, 16, 64, "dense"),
    _edge("edge_seqlens_bf16", "fmha_bf16_seqlens_edge", "bf16", 65535, 2, 1, 16, 64, "seqlens"),
    _edge("edge_paged_f16", "fmha_f16_paged_edge", "f16", 65535, 2, 1, 16, 64, "paged"),
    _edge("edge_varlen_f16", "fmha_f16_varlen_edge", "f16", 65535, 1, 1, 16, 64, "varlen"),
    _hgemm("hgemm_f16_nn", "hgemm_f16", 47104, 47104, 64),
    _hgemm("hgemm_f16acc_tn", "hgemm_f16acc", 47104, 47104, 64, acc="f16", tn=True),
    _hgemm("hgemm_f16_rows", "hgemm_f16_rows", 47104, 47104, 64, rows=1024),
    _sgemm("sgemm_tf32_nn", "sgemm_tf32_nn", 47104, 47104, 64, "tf32"),
    _sgemm("sgemm_tf32_tn", "sgemm_tf32_tn", 47104, 47104, 64, "tf32", tn=True),
    _sgemm("sgemm_3xtf32", "sgemm_3xtf32", 47104, 47104, 64, "3xtf32"),
    _sgemm("sgemm_tf32_nn_k2097216", "sgemm_tf32_nn_longk", 64, 64, 2_097_216, "tf32", gen="ternary"),
    _sgemm("sgemm_tf32_nn_noround_k2097216", "sgemm_tf32_nn_noround_longk", 64, 64, 2_097_216, "tf32", rnd=False,
           gen="ternary"),
    _sgemm("sgemm_tf32_nn_k2097216_tail", "sgemm_tf32_nn_longk", 64, 64, 2_097_216, "tf32", gen="tail"),
    _sgemm("sgemm_3xtf32_k2097216", "sgemm_3xtf32_longk", 64, 64, 2_097_216, "3xtf32", gen="ternary"),
    _sgemm("sgemm_tf32_nn_k2097120", "sgemm_tf32_nn_kedge", 64, 64, 2_097_120, "tf32", gen="ternary"),
    _merge("merge_f16", "f16", 1_048_704, 16, 128, False),
    _merge("merge_bf16", "bf16", 1_048_704, 16, 128, False),
    _merge("merge_f32_in_place", "f32", 1_048_704, 16, 128, True),
    _rows("rope_f32_in_place", "rope_f32", "f32", 8_388_609, 256, True),
    _rope_qk("rope_qk_in_place", 1, 32, 524_289, 128),
    _rows("rms_norm_f16", "rms_norm_f16", "f16", 2_097_153, 1024, False),
    _rows("rms_norm_f32", "rms_norm_f32", "f32", 2_097_153, 1024, False),
    _rows("tf32_round_in_place", "tf32_round", "f32", 16_777_344, 128, True),
]

# The sgemm cases whose K passes 65535 k-tiles of 32, the grid limit of the TF32 transpose before it looped over k-tiles.
TRANSPOSE_K_LIMIT = 65535 * 32


def by_name(cases=None):
    return {c.name: c for c in (CASES if cases is None else cases)}
