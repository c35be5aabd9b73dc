/* leetcuda_b200.h — C ABI of the H100-native (sm_90a) replacement for LeetCUDA's
 * two dense-contraction hot paths.  Plain pointers and sizes only: no torch
 * types cross this boundary.  All device pointers must live on the CUDA device
 * that is current on the calling thread; `stream` is a cudaStream_t (NULL = the
 * legacy default stream, which is what the reference launches on).
 *
 * Every entry point returns 0 on success or a negative B200_E* code; the text of
 * the last failure on the calling thread is returned by b200_last_error().
 * The reference's ops throw std::runtime_error for the same conditions
 * (kernels/hgemm/utils/utils.h:137-147, kernels/flash-attn/utils/utils.h) and
 * never check CUDA errors; the Python mirror in leetcuda_b200/ turns a non-zero
 * status into RuntimeError so callers see the reference's behaviour.
 */
#ifndef LEETCUDA_B200_H_
#define LEETCUDA_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200_OK 0
#define B200_EINVAL (-1)  /* bad shape / alignment / null pointer            */
#define B200_ECUDA (-2)   /* CUDA runtime or driver error (text in last_error) */
#define B200_ENOTSUP (-3) /* e.g. head dim outside the dispatch set          */

/* Layout of the B operand of b200_hgemm_f16. */
#define B200_B_ROW_MAJOR_KN 0 /* "NN": b is [K,N] row-major (N contiguous)           */
#define B200_B_ROW_MAJOR_NK 1 /* "TN": b storage is [N,K] row-major (K contiguous)   */

/* ABI version of this header (major*1000 + minor). */
int b200_version(void);

/* Text of the last error raised on the calling thread ("" if none). */
const char* b200_last_error(void);

/* Number of kernels this library has launched in the calling process (all
 * threads).  Used by bench.py to report `gpu_launches`. */
uint64_t b200_launch_count(void);

/* C[M,N] = A[M,K] x B, fp16 in / fp16 out, fp32 accumulation (wgmma, registers).
 *
 * Replaces every `void hgemm_*(torch::Tensor a, torch::Tensor b, torch::Tensor c
 * [, int stages, bool swizzle, int swizzle_stride])` bound in the reference's
 * kernels/hgemm/pybind/hgemm.cc:124-182 (host launchers e.g.
 * kernels/hgemm/mma/swizzle/hgemm_mma_stage_swizzle.cu:808-887 for NN and
 * kernels/hgemm/mma/basic/hgemm_mma_stage_tn.cu:555-629 for TN).  The reference's
 * stages/swizzle/swizzle_stride arguments are tuning hints of its own tiling and
 * have no counterpart here.
 *
 * a: [M,K] row-major.  b: see b_layout.  c: [M,N] row-major, written in place.
 * Constraints: M,N,K > 0; K % 8 == 0 and N % 8 == 0 (16-byte TMA strides);
 * pointers 16-byte aligned.  Unlike the reference (M,N % 128 == 0, K % 32 == 0,
 * hgemm_mma_stage.cu:675-676) ragged M/N/K tiles are handled.
 */
int b200_hgemm_f16(const void* a, const void* b, void* c, int M, int N, int K, int b_layout,
                   void* stream);

/* Reference-accumulation parity mode: same as b200_hgemm_f16 but the tensor core accumulates in
 * fp16 (wgmma D format f16, one rounding per k16 instruction) exactly like the reference's
 * HMMA.16816.F16 kernels (mma/basic/hgemm_mma.cu:67-73) and its cuBLAS CUBLAS_COMPUTE_16F op
 * (cublas/hgemm_cublas.cu:50-52).  Less accurate than the default fp32 accumulation; provided so
 * that outputs can be compared with the reference's bit for bit.  Select it for every mirror op
 * with LEETCUDA_B200_HGEMM_ACC=f16. */
int b200_hgemm_f16_acc16(const void* a, const void* b, void* c, int M, int N, int K, int b_layout,
                         void* stream);

/* Row-sharded variant used by the multi-GPU path (SURVEY.md §8e): computes the
 * rows [row0, row0+rows) of C = A_shard x B where a_shard is [rows,K] and writes
 * them into c_full (an [M_total,N] buffer) at row offset row0.  c_full may be a
 * peer-mapped pointer of another GPU (NVLink P2P store from the epilogue). */
int b200_hgemm_f16_rows(const void* a_shard, const void* b, void* c_full, int rows, int N, int K,
                        int b_layout, int row0, void* stream);

/* Fused GEMM + all-gather of C: like b200_hgemm_f16_rows, but the epilogue also delivers every
 * finished tile to the other GPUs while the remaining tiles are still being computed.  At least one
 * of the two target descriptions must be given (else B200_EINVAL):
 *   c_full_peers / n_peers (1..7) : peer-mapped C buffers of the other GPUs.  This is the default
 *                              transport: the epilogue stores every value to c_full and to every
 *                              peer (NVLink P2P).
 *   c_full_multicast         : an NVLS multicast mapping of the symmetric C buffer.  Used when no
 *                              peers are given (one multimem.st reaches every GPU, this one
 *                              included), or when B200_FUSED_EPILOGUE=direct|mc selects it.
 * n_peers > 0 with c_full_peers == NULL is rejected.  The caller closes the step with a cross-GPU
 * barrier and must not let a peer overwrite a C buffer that is still being read (leetcuda_b200/dist.py
 * alternates two symmetric buffers). */
int b200_hgemm_f16_rows_fused(const void* a_shard, const void* b, void* c_full, void* c_full_multicast,
                              void* const* c_full_peers, int n_peers, int rows, int N, int K,
                              int b_layout, int row0, void* stream);

/* O = softmax(Q K^T * scale) V per (batch, head); fp16 in/out, fp32 softmax
 * statistics and fp32 accumulation; non-causal, no mask, no dropout.
 *
 * Replaces every `void flash_attn_mma_stages_*(Q,K,V,O,int stages)` bound in
 * kernels/flash-attn/pybind/flash_attn.cc:168-224 (e.g. the shared-QKV launcher
 * kernels/flash-attn/mma/basic/flash_attn_mma_share_qkv.cu:770-921), the CuTe op
 * flash_attn_cute (cutlass/flash_attn_cute.cu:496-524) and ffpa-attn's
 * ffpa_mma_acc_{f16,f32}_L1 (ffpa-attn/csrc/pybind/ffpa_attn_api.cc:8-16).
 *
 * q,k,o: [B,H,N,D] contiguous.  v: [B,H,N,D] (v_transposed = 0) or [B,H,D,N]
 * (v_transposed = 1, the reference's *_swizzle_qkv ops).  scale <= 0 selects the
 * reference's 1/sqrt(D) (flash_attn_mma_split_q.cu:79).
 * Constraints: D % 8 == 0 and D <= 1024; any N >= 1 (N % 8 == 0 for v_transposed).  For
 * v_transposed with D > 128 V is first restored to [B,H,N,D] in a stream-ordered scratch
 * allocation (cudaMallocAsync / cudaFreeAsync on `stream`).
 * Kernel (wgmma, TMA, mbarrier): each CTA owns a query tile and a column slab of O — one slab of 64 / 128
 * columns for D <= 64 / D <= 128, 256-column slabs above (each slab recomputes S).
 * Numerics: S, the softmax statistics and O in fp32, P rounded to fp16 before P.V (as the reference); the
 * exponentials are ex2.approx (MUFU) except, for D <= 128, a fixed quarter of the keys, which a degree-3 polynomial on
 * the FMA pipe evaluates with max. relative error 7.6e-5 — below the fp16 rounding P receives next
 * (tests/test_softmax_math.py).  Tolerance against the reference: allclose(1e-2, 1e-2), its own criterion.
 */
int b200_fmha_fwd_f16(const void* q, const void* k, const void* v, void* o, int B, int H, int N,
                      int D, int v_transposed, float scale, void* stream);

/* Same, and also writes lse[b,h,i] = ln sum_j exp(scale * q_i . k_j) (fp32, [B,H,N] contiguous):
 * the per-row statistic that b200_merge_attn_states consumes (as [num_heads, num_tokens] when B = 1)
 * to combine partial results over disjoint key ranges (split-KV).  The reference's attention ops
 * have no such output (its merge test feeds synthetic LSEs,
 * kernels/openai-triton/merge-attn-states/test_merge_attn_states.py:100-152). */
int b200_fmha_fwd_f16_lse(const void* q, const void* k, const void* v, void* o, float* lse, int B,
                          int H, int N, int D, int v_transposed, float scale, void* stream);

/* Attention with separate query and key lengths and an optional causal mask: prefill against a KV cache, decoding
 * (Nq << Nk), cross-attention, and the parts of a split-KV computation that b200_merge_attn_states combines.
 *
 * q, o: [B,H,Nq,D] contiguous.  k: [B,H,Nk,D].  v: [B,H,Nk,D] (v_transposed = 0) or [B,H,D,Nk] (v_transposed = 1).
 * lse: [B,H,Nq] fp32, ln sum_j exp(scale * q_i . k_j) over the visible keys, or NULL.  scale <= 0 selects 1/sqrt(D).
 * causal = 1 masks key j for query i when j > i + (Nk - Nq): the diagonal is aligned bottom-right, as in
 * FlashAttention-2, so the Nq queries are the last Nq positions of a sequence whose first Nk - Nq keys come from a
 * cache; with Nq = Nk it is the usual lower triangle.  This is NOT torch SDPA's is_causal when Nq != Nk: SDPA aligns
 * the diagonal top-left (key j masked when j > i).  With Nq > Nk the rows i < Nq - Nk see no key; such an empty row
 * gets O = 0 and lse = -inf (never NaN), which b200_merge_attn_states treats as a part without keys.
 * causal = 0 with Nq = Nk computes exactly what b200_fmha_fwd_f16_lse / b200_fmha_fwd_f16 compute.
 * Constraints: Nq, Nk >= 1; causal is 0 or 1; D % 8 == 0 and D <= 1024; B * H <= 65535; Nk % 8 == 0 for
 * v_transposed (for D > 128 V is first restored to [B,H,Nk,D] in stream-ordered scratch, as above).  Numerics as for
 * b200_fmha_fwd_f16.  A causal CTA visits only the key blocks left of its diagonal, about half the work at Nq = Nk. */
int b200_fmha_fwd_f16_kv(const void* q, const void* k, const void* v, void* o, float* lse /* may be NULL */,
                         int B, int H, int Nq, int Nk, int D, int v_transposed, int causal, float scale, void* stream);

/* Grouped-query attention (GQA / MQA) and split-KV decoding: b200_fmha_fwd_f16_kv with fewer K/V heads than query heads,
 * and the keys of every CTA optionally cut into num_splits ranges that run in parallel.
 *
 * q, o: [B,H,Nq,D] contiguous.  k: [B,Hkv,Nk,D].  v: [B,Hkv,Nk,D] (v_transposed = 0) or [B,Hkv,D,Nk] (v_transposed = 1).
 * lse: [B,H,Nq] fp32 or NULL.  H % Hkv == 0; query head h reads K/V head h / (H / Hkv), the convention of torch SDPA's
 * enable_gqa and of FlashAttention.  Hkv == H is multi-head and Hkv == 1 multi-query attention.  Causal masking, empty
 * rows (O = 0, lse = -inf), scale, lse and numerics are those of b200_fmha_fwd_f16_kv.  The H / Hkv query heads of a
 * K/V head run as one tile of packed rows, so each K/V block is read once per group and a decode step fills
 * H / Hkv rows of the tile instead of one.
 * num_splits = 1: no split, one launch (with transposed V and D > 128 the pre-pass is a second one), and O, lse equal
 * those of b200_fmha_fwd_f16_kv on K and V with every head repeated H / Hkv times, bit for bit.  num_splits = n > 1:
 * the key blocks each CTA visits are cut into n contiguous ranges (a range may be empty and then contributes nothing);
 * every split writes its normalised O in fp32 and its lse to a stream-ordered workspace (cudaMallocAsync /
 * cudaFreeAsync on `stream`, (n * B * H * Nq * (D + 1)) * 4 bytes), and a second launch combines the parts with their
 * lse weights and rounds once to fp16.  num_splits = 0 lets the library choose from the shapes and the SM count: 1 when
 * the unsplit grid already fills the GPU, otherwise enough splits to cover the SMs once — the choice for decoding.
 * Constraints: those of b200_fmha_fwd_f16_kv, with the grid limit on B * Hkv <= 65535 instead of B * H;
 * Hkv >= 1 and H % Hkv == 0; 0 <= num_splits <= B200_FMHA_MAX_SPLITS; with num_splits != 1, o 16-byte aligned (the
 * combine stores 16-byte packs; a tensor from a CUDA allocator is). */
#define B200_FMHA_MAX_SPLITS 64
int b200_fmha_fwd_f16_gqa(const void* q, const void* k, const void* v, void* o, float* lse /* may be NULL */,
                          int B, int H, int Hkv, int Nq, int Nk, int D, int v_transposed, int causal,
                          int num_splits, float scale, void* stream);

/* The split count b200_fmha_fwd_f16_gqa chooses for num_splits = 0 on the current device (>= 1), or a negative
 * B200_E* code for a bad shape.  Depends on the shapes and the device's SM count only (not on causal or the layout). */
int b200_fmha_fwd_f16_gqa_splits(int B, int H, int Hkv, int Nq, int Nk, int D);

/* Per-sequence query and key lengths over padded buffers: batched decoding and prefill against a KV cache.
 *
 * q, o: [B,H,Nq,D].  k, v: [B,Hkv,Nk,D] (natural V only), e.g. a KV cache allocated for Nk positions.  lse: [B,H,Nq]
 * fp32 or NULL.  seqlens_q, seqlens_k: int32 [B] in device memory, or NULL for Nq resp. Nk for every sequence.
 * Sequence b has Lq_b = clamp(seqlens_q[b], 0, Nq) queries (rows 0 .. Lq_b - 1) and Lk_b = clamp(seqlens_k[b], 0, Nk)
 * keys (rows 0 .. Lk_b - 1).  Keys at or past Lk_b contribute nothing whatever they hold (NaN, Inf, stale data); causal
 * masking is per sequence and bottom-right: key j is masked for query i when j > i + (Lk_b - Lq_b).  Padded rows
 * (i >= Lq_b) and rows without a visible key get O = 0 and lse = -inf, written as such even where Q holds NaN, so the
 * output holds no uninitialised memory and b200_merge_attn_states treats those rows as empty parts.
 * The lengths are read by the kernel only: the host neither copies them nor synchronises, so a captured CUDA graph
 * replays correctly after new lengths are written into the same arrays.  num_splits = 0 chooses the split count from
 * the padded shape (b200_fmha_fwd_f16_gqa_splits(B, H, Hkv, Nq, Nk, D)), not from the lengths.  GQA head mapping,
 * scale, num_splits, the split workspace, the combine and numerics are those of b200_fmha_fwd_f16_gqa; with
 * num_splits = 1 each sequence's rows equal b200_fmha_fwd_f16_gqa on that sequence alone (Nq = Lq_b, Nk = Lk_b), bit
 * for bit.  Constraints: those of b200_fmha_fwd_f16_gqa (B * Hkv <= 65535, o 16-byte aligned when num_splits != 1),
 * and the length arrays 4-byte aligned with B entries. */
int b200_fmha_fwd_f16_seqlens(const void* q, const void* k, const void* v, void* o, float* lse /* may be NULL */,
                              const int* seqlens_q /* may be NULL */, const int* seqlens_k /* may be NULL */,
                              int B, int H, int Hkv, int Nq, int Nk, int D, int causal, int num_splits, float scale,
                              void* stream);

/* Paged KV cache: b200_fmha_fwd_f16_seqlens with K and V kept in a pool of fixed-size pages and a block table per
 * sequence (the layout of FlashAttention's block-table API and of vLLM's flash-attn backend).
 *
 * q, o: [B,H,Nq,D].  k_cache, v_cache: each [num_pages, page_size, Hkv, D] fp16, contiguous.  block_table: int32
 * [B, max_pages_per_seq], contiguous, in device memory.  Key t of sequence b is row t % page_size of page
 * block_table[b][t / page_size].  Everything else is b200_fmha_fwd_f16_seqlens with the padded
 * Nk = max_pages_per_seq * page_size: the length clamps, the per-sequence bottom-right causal mask, O = 0 and
 * lse = -inf in padded rows and rows without a key, the GQA mapping, num_splits (0 chooses from the padded shape),
 * the split workspace, the combine and the numerics.  With the same data, O and lse equal those of
 * b200_fmha_fwd_f16_seqlens on a contiguous padded cache, bit for bit.
 * Table entries at or past a sequence's last used page, ceil(Lk_b / page_size), are never read: callers may pad the
 * table with -1 or stale ids.  Pages may be shared between sequences (prefix sharing); the pool is only read.  A page
 * id is only ever a TMA coordinate, bounds-checked against the pool: a used entry outside [0, num_pages) gives wrong
 * values for that sequence, never an out-of-bounds access.  The table and the lengths are read by the kernel only, so
 * a captured CUDA graph replays correctly after new tables or lengths are written into the same arrays.
 * Constraints: those of b200_fmha_fwd_f16_seqlens; page_size a power of two >= 16; num_pages >= 1,
 * max_pages_per_seq >= 1; num_pages * page_size and max_pages_per_seq * page_size <= 2^31 - 1; block_table 4-byte
 * aligned. */
int b200_fmha_fwd_f16_paged(const void* q, const void* k_cache, const void* v_cache, void* o,
                            float* lse /* may be NULL */, const int* block_table,
                            const int* seqlens_q /* may be NULL */, const int* seqlens_k /* may be NULL */, int B,
                            int H, int Hkv, int Nq, int num_pages, int page_size, int max_pages_per_seq, int D,
                            int causal, int num_splits, float scale, void* stream);

/* bf16 attention: b200_fmha_fwd_f16_seqlens and b200_fmha_fwd_f16_paged with q, k, v (k_cache, v_cache) and o in
 * bf16.  Argument lists, constraints, error codes and messages, and semantics are those of the f16 entries: the length
 * clamps, the per-sequence bottom-right causal mask, O = 0 and lse = -inf in padded rows and rows without a key, the
 * GQA mapping, num_splits (0 chooses b200_fmha_fwd_f16_gqa_splits(B, H, Hkv, Nq, Nk, D), which does not depend on
 * the element type), the split workspace and its combine, and the lengths and tables read on the GPU only.  lse stays
 * fp32.  NULL seqlens_q and seqlens_k give the dense call (one length Nq / Nk for every sequence, MHA or GQA, causal
 * or not, split or not).  The element type is the only difference: S and O accumulate in fp32 as for fp16, P is
 * rounded to bf16 (nearest even) before P V, and O is rounded once to bf16.  bf16 has fp32's exponent range, so
 * inputs and outputs beyond fp16's 65504 are fine.  Natural V only, as for the f16 entries. */
int b200_fmha_fwd_bf16_seqlens(const void* q, const void* k, const void* v, void* o, float* lse /* may be NULL */,
                               const int* seqlens_q /* may be NULL */, const int* seqlens_k /* may be NULL */,
                               int B, int H, int Hkv, int Nq, int Nk, int D, int causal, int num_splits, float scale,
                               void* stream);
/* fp8 (OCP e4m3, torch.float8_e4m3fn) K and V with fp16 or bf16 q and o: the argument lists of
 * b200_fmha_fwd_{f16,bf16}_seqlens and _paged plus k_scale and v_scale before stream; k, v (k_cache, v_cache) hold
 * e4m3 bytes, [B, Hkv, Nk, D] resp. pools [num_pages, page_size, Hkv, D].  O = softmax(scale * Q (k_scale K)^T)
 * (v_scale V) with every semantic of the counterpart (lengths, causal mask, GQA, split-KV, paging, padded rows).
 * K and V are widened exactly to the type of q; k_scale is folded into the softmax scale as fp32(scale * k_scale)
 * (scale <= 0 is first replaced by 1/sqrt(D)), and v_scale multiplies the normalised fp32 O (or each split's part)
 * before O's one rounding; lse does not see v_scale.  With v_scale = 1 the call is bit for bit the counterpart on
 * K and V converted to q's type with scale = fp32(scale * k_scale).
 * Checks: exactly those of the counterpart with its codes and messages, then B200_EINVAL for D % 16 != 0 (an e4m3 row
 * of D bytes is the TMA row stride), for k_scale or v_scale not finite and > 0, and for fp32(scale * k_scale) not
 * finite and > 0. */
int b200_fmha_fwd_f16_fp8kv_seqlens(const void* q, const void* k, const void* v, void* o, float* lse /* may be NULL */,
                                    const int* seqlens_q /* may be NULL */, const int* seqlens_k /* may be NULL */,
                                    int B, int H, int Hkv, int Nq, int Nk, int D, int causal, int num_splits,
                                    float scale, float k_scale, float v_scale, void* stream);
int b200_fmha_fwd_bf16_fp8kv_seqlens(const void* q, const void* k, const void* v, void* o, float* lse /* may be NULL */,
                                     const int* seqlens_q /* may be NULL */, const int* seqlens_k /* may be NULL */,
                                     int B, int H, int Hkv, int Nq, int Nk, int D, int causal, int num_splits,
                                     float scale, float k_scale, float v_scale, void* stream);
int b200_fmha_fwd_f16_fp8kv_paged(const void* q, const void* k_cache, const void* v_cache, void* o,
                                  float* lse /* may be NULL */, const int* block_table,
                                  const int* seqlens_q /* may be NULL */, const int* seqlens_k /* may be NULL */, int B,
                                  int H, int Hkv, int Nq, int num_pages, int page_size, int max_pages_per_seq, int D,
                                  int causal, int num_splits, float scale, float k_scale, float v_scale, void* stream);
int b200_fmha_fwd_bf16_fp8kv_paged(const void* q, const void* k_cache, const void* v_cache, void* o,
                                   float* lse /* may be NULL */, const int* block_table,
                                   const int* seqlens_q /* may be NULL */, const int* seqlens_k /* may be NULL */,
                                   int B, int H, int Hkv, int Nq, int num_pages, int page_size, int max_pages_per_seq,
                                   int D, int causal, int num_splits, float scale, float k_scale, float v_scale,
                                   void* stream);
int b200_fmha_fwd_bf16_paged(const void* q, const void* k_cache, const void* v_cache, void* o,
                             float* lse /* may be NULL */, const int* block_table,
                             const int* seqlens_q /* may be NULL */, const int* seqlens_k /* may be NULL */, int B,
                             int H, int Hkv, int Nq, int num_pages, int page_size, int max_pages_per_seq, int D,
                             int causal, int num_splits, float scale, void* stream);

/* Packed variable-length attention (FlashAttention's flash_attn_varlen_func layout): the tokens of B sequences packed
 * one after the other, no padding.
 *
 * q, o: [total_q, H, D].  k, v: [total_k, Hkv, D].  lse: fp32 [H, total_q] or NULL (the layout of
 * b200_merge_attn_states' lse).  cu_seqlens_q, cu_seqlens_k: int32 [B + 1] in device memory.  Sequence b has
 * Lq_b = clamp(cu_seqlens_q[b+1] - cu_seqlens_q[b], 0, max_seqlen_q) queries at rows cu_seqlens_q[b] + t and
 * Lk_b = clamp(cu_seqlens_k[b+1] - cu_seqlens_k[b], 0, max_seqlen_k) keys at rows cu_seqlens_k[b] + t.  Query head h
 * reads K/V head h / (H / Hkv).  Causal masking is per sequence and bottom-right: key j is masked for query i when
 * j > i + (Lk_b - Lq_b); a row without a visible key (Lk_b = 0 included) gets O = 0 and lse = -inf.
 * Only rows cu_seqlens_q[b] + t with t < Lq_b and 0 <= cu_seqlens_q[b] + t < total_q are written: rows of o and
 * columns of lse that no sequence owns keep their contents, whatever the arrays hold (bad offsets give wrong values,
 * never an out-of-bounds store; loads are bounds-checked TMA coordinates).  Keys of the next sequence in the last
 * partial key block of sequence b contribute nothing, whatever they hold.  The offsets are read by the kernel only
 * (no host copy, no synchronisation), so a captured CUDA graph replays with new offsets written into the same arrays.
 * Numerics: O and lse are those of b200_fmha_fwd_f16_seqlens with num_splits = 1 on padded [B,H,max_seqlen_q,D] /
 * [B,Hkv,max_seqlen_k,D] copies of the same data, bit for bit.  One launch, no workspace, no split.
 * Every query head gets ceil(max_seqlen_q / 128) tiles of its own (of 64 rows for D > 128): a batch of one-token
 * decode rows runs at 1/128 of the tile's rows; decoding should use the seqlens or paged entries.
 * Constraints: B, H, D, total_q, total_k, max_seqlen_q, max_seqlen_k >= 1; Hkv >= 1 divides H; B * Hkv <= 65535;
 * (H / Hkv) * max_seqlen_q <= 2^31 - 1 and the grid's (H / Hkv) * ceil(max_seqlen_q / 128) * slabs CTAs as well;
 * total_q * H * D and total_k * Hkv * D addressable; the offset arrays 4-byte aligned; D % 8 == 0 and D <= 1024
 * (B200_ENOTSUP otherwise).  scale <= 0 means 1/sqrt(D).  bf16: the same entry with bf16 q, k, v and o. */
int b200_fmha_fwd_f16_varlen(const void* q, const void* k, const void* v, void* o, float* lse /* may be NULL */,
                             const int* cu_seqlens_q, const int* cu_seqlens_k, int B, int H, int Hkv, int total_q,
                             int total_k, int max_seqlen_q, int max_seqlen_k, int D, int causal, float scale,
                             void* stream);
int b200_fmha_fwd_bf16_varlen(const void* q, const void* k, const void* v, void* o, float* lse /* may be NULL */,
                              const int* cu_seqlens_q, const int* cu_seqlens_k, int B, int H, int Hkv, int total_q,
                              int total_k, int max_seqlen_q, int max_seqlen_k, int D, int causal, float scale,
                              void* stream);

/* Packed queries against a paged KV cache (vLLM's chunked prefill): b200_fmha_fwd_f16_varlen with k_cache, v_cache
 * pools [num_pages, page_size, Hkv, D] and block_table int32 [B, max_pages_per_seq] as in b200_fmha_fwd_f16_paged.
 * Sequence b has Lk_b = clamp(seqused_k[b], 0, max_pages_per_seq * page_size) keys (seqused_k: int32 [B] in device
 * memory); key t is row t % page_size of page block_table[b][t / page_size].  Every other rule is the packed rule.
 * Numerics: bit for bit b200_fmha_fwd_f16_paged with num_splits = 1 on a padded copy of q.  Constraints: those of the
 * packed entry without total_k / max_seqlen_k, and the paged constraints of b200_fmha_fwd_f16_paged. */
int b200_fmha_fwd_f16_varlen_paged(const void* q, const void* k_cache, const void* v_cache, void* o,
                                   float* lse /* may be NULL */, const int* cu_seqlens_q, const int* seqused_k,
                                   const int* block_table, int B, int H, int Hkv, int total_q, int max_seqlen_q,
                                   int num_pages, int page_size, int max_pages_per_seq, int D, int causal,
                                   float scale, void* stream);
int b200_fmha_fwd_bf16_varlen_paged(const void* q, const void* k_cache, const void* v_cache, void* o,
                                    float* lse /* may be NULL */, const int* cu_seqlens_q, const int* seqused_k,
                                    const int* block_table, int B, int H, int Hkv, int total_q, int max_seqlen_q,
                                    int num_pages, int page_size, int max_pages_per_seq, int D, int causal,
                                    float scale, void* stream);

/* ------------------------------------------------------------------ KV-cache append
 * The write half of a decode or chunked-prefill step, in one launch (FlashAttention's flash_attn_with_kvcache append,
 * vLLM's reshape_and_cache_flash): rotate q and the new k at each sequence's own positions, quantise k and v when the
 * cache is e4m3, and scatter the new tokens into a dense or paged cache.  The attention call that follows takes
 * seqlens_k = seqlens_out (b200_fmha_fwd_*_seqlens / _paged / _fp8kv_*).
 *
 * k_new, v_new: [B, Hkv, n_new, D] of T (f16 entries: fp16, bf16 entries: bf16).  cache_seqlens: int32 [B] in device
 * memory.  Sequence b holds L_b = clamp(cache_seqlens[b], 0, capacity) tokens; new token t goes to position
 * p = L_b + t, where capacity = Nk (dense) or max_pages_per_seq * page_size (paged).
 *   dense: k_cache, v_cache [B, Hkv, Nk, D] (the layout of b200_fmha_fwd_f16_seqlens); row p of (b, h).
 *   paged: pools [num_pages, page_size, Hkv, D] and block_table int32 [B, max_pages_per_seq] (the layout of
 *          b200_fmha_fwd_f16_paged); row p % page_size of page block_table[b][p / page_size].  A table entry outside
 *          [0, num_pages) means the token is not written.
 * Tokens with p >= capacity are dropped; nothing is ever written out of bounds.  Every other cache byte keeps its value.
 * cache_dtype: T's B200_DTYPE_F16 / B200_DTYPE_BF16 (the cache is T), or B200_DTYPE_E4M3: the cache holds
 * cvt.rn.satfinite.e4m3(float(x) / scale) of the T value x (after rotary), an IEEE division, k_scale for k and v_scale
 * for v — bit for bit torch's (x.float() / scale).clamp(-448, 448).to(torch.float8_e4m3fn).  The scales are per tensor,
 * finite and > 0, and exactly 1 unless the cache is e4m3.
 * seqlens_out (may be NULL): int32 [B], receives min(L_b + n_new, capacity), the key lengths of the attention call.
 * q, q_out (both NULL or both set): [B, H, n_new, D] of T; q_out receives q rotated at the same positions p (every
 * token, dropped or not); q_out == q rotates in place.  Without rotary tables q is copied.
 * rotary_cos, rotary_sin (both NULL or both set): fp32 [rotary_len, rotary_dim / 2], indexed [p, i].  Pair i is
 * (2i, 2i+1) with rotary_interleaved = 1 (GPT-J) and (i, i + rotary_dim / 2) with 0 (NeoX / Llama);
 * x0' = x0 c - x1 s, x1' = x0 s + x1 c in fp32, rounded once to T; columns >= rotary_dim are copied; v is never rotated.
 * Without tables rotary_dim, rotary_len and rotary_interleaved must be 0.
 * Lengths and tables are read by the kernel only (no host copy, no synchronisation): a captured CUDA graph replays with
 * the lengths the arrays hold at replay time.  Two sequences that write the same row of a shared page race; the
 * library does not detect it.
 * Checks (B200_EINVAL, message naming the argument, before any CUDA call): pointers; B, H, Hkv, n_new, D, Nk
 * (num_pages, page_size, max_pages_per_seq) >= 1; H % Hkv == 0; cache_dtype; D % 8 == 0 (D % 16 == 0 for e4m3);
 * page_size a power of two >= 16; capacity + n_new <= 2^31 - 1 and B * n_new * (2 Hkv + H) <= 2^31 - 1;
 * rotary_dim % 16 == 0 and 0 < rotary_dim <= D; rotary_len >= capacity + n_new (positions come from device memory);
 * the scales; tensors 16-byte aligned, int arrays 4-byte aligned; every buffer the call writes (k_cache, v_cache,
 * q_out unless it is q, seqlens_out) disjoint from every other buffer.  One launch. */
int b200_kvcache_append_f16(const void* k_new, const void* v_new, void* k_cache, void* v_cache,
                            const int* cache_seqlens, int* seqlens_out /* may be NULL */, const void* q /* may be NULL */,
                            void* q_out /* may be NULL */, const float* rotary_cos /* may be NULL */,
                            const float* rotary_sin /* may be NULL */, int B, int H, int Hkv, int n_new, int Nk, int D,
                            int rotary_dim, int rotary_len, int rotary_interleaved, int cache_dtype, float k_scale,
                            float v_scale, void* stream);
int b200_kvcache_append_bf16(const void* k_new, const void* v_new, void* k_cache, void* v_cache,
                             const int* cache_seqlens, int* seqlens_out /* may be NULL */, const void* q /* may be NULL */,
                             void* q_out /* may be NULL */, const float* rotary_cos /* may be NULL */,
                             const float* rotary_sin /* may be NULL */, int B, int H, int Hkv, int n_new, int Nk, int D,
                             int rotary_dim, int rotary_len, int rotary_interleaved, int cache_dtype, float k_scale,
                             float v_scale, void* stream);
int b200_kvcache_append_f16_paged(const void* k_new, const void* v_new, void* k_cache, void* v_cache,
                                  const int* block_table, const int* cache_seqlens, int* seqlens_out /* may be NULL */,
                                  const void* q /* may be NULL */, void* q_out /* may be NULL */,
                                  const float* rotary_cos /* may be NULL */, const float* rotary_sin /* may be NULL */,
                                  int B, int H, int Hkv, int n_new, int num_pages, int page_size, int max_pages_per_seq,
                                  int D, int rotary_dim, int rotary_len, int rotary_interleaved, int cache_dtype,
                                  float k_scale, float v_scale, void* stream);
int b200_kvcache_append_bf16_paged(const void* k_new, const void* v_new, void* k_cache, void* v_cache,
                                   const int* block_table, const int* cache_seqlens, int* seqlens_out /* may be NULL */,
                                   const void* q /* may be NULL */, void* q_out /* may be NULL */,
                                   const float* rotary_cos /* may be NULL */, const float* rotary_sin /* may be NULL */,
                                   int B, int H, int Hkv, int n_new, int num_pages, int page_size,
                                   int max_pages_per_seq, int D, int rotary_dim, int rotary_len, int rotary_interleaved,
                                   int cache_dtype, float k_scale, float v_scale, void* stream);

/* ------------------------------------------------------------------ SGEMM (TF32)
 * C[M,N] (fp32) = A[M,K] (fp32) x B on the tensor cores through wgmma .tf32 with fp32
 * accumulation — the sibling of the HGEMM path (SURVEY §8f-2).  Replaces
 *   sgemm_wmma_m16n16k8_mma4x2_warp2x4_stages{,_dsmem}(a,b,c,stages,swizzle,swizzle_stride)
 *   (kernels/sgemm/sgemm_wmma_tf32_stage.cu:573-742, bound in kernels/sgemm/sgemm.cu:762-764).
 * Like the reference (sgemm_wmma_tf32_stage.cu:586-592: f32x4_tf32x4_kernel over a and b IN PLACE),
 * round_inputs_in_place != 0 first rewrites a and b with their TF32 roundings (cvt.rna.tf32.f32);
 * with 0 the inputs are left untouched and the tensor core reads the upper 19 bits of each fp32
 * (truncation).  b_layout as for b200_hgemm_f16 (the reference has only the [K,N] form).
 * Constraints: M,N,K > 0; K % 4 == 0 and N % 4 == 0; pointers 16-byte aligned.
 */
int b200_sgemm_tf32(float* a, float* b, float* c, int M, int N, int K, int b_layout,
                    int round_inputs_in_place, void* stream);

/* fp32 product on the TF32 tensor cores through the 3xTF32 split: every operand is split into two TF32 numbers
 * (x = hi + lo, both exactly representable) and C = hi_a hi_b + hi_a lo_b + lo_a hi_b is evaluated by ONE tf32 GEMM
 * over concatenated operands (K' = 3K, scratch from cudaMallocAsync on `stream`).  The operand rounding of a plain
 * TF32 product (1e-3 relative) is gone; what remains is the tensor core's truncating fp32 accumulation: measured
 * 5e-5 relative at K = 1024..4096, against 2e-6 for an FFMA kernel.  That is why the reference's 13 CUDA-core fp32
 * ops (kernels/sgemm/sgemm.cu:743-760, kernels/sgemm/sgemm_async.cu) stay vendor fp32 rows in the Python mirror by
 * default and use this entry only under LEETCUDA_B200_SGEMM_FP32=3xtf32.
 * a: [M,K], b: [K,N], c: [M,N] row-major fp32; a and b are not modified.  K % 4 == 0, N % 4 == 0. */
int b200_sgemm_3xtf32(const float* a, const float* b, float* c, int M, int N, int K, void* stream);

/* x[i] <- tf32(x[i]) (round to nearest, ties away), in place, n elements; x 16-byte aligned. */
int b200_tf32_round_inplace(float* x, size_t n, void* stream);

/* ------------------------------------------------------------------ fp8 (e4m3) scaled GEMM
 * C[M,N] = OutT( scaled( A[M,K] B[N,K]^T ) ): A and B OCP e4m3 (torch.float8_e4m3fn), both K-major; C fp16 or bf16
 * (c_dtype B200_DTYPE_F16 / B200_DTYPE_BF16), row-major, written in place.  The layout of torch's _scaled_mm with a
 * column-major [K,N] b, i.e. a [N,K] row-major weight.
 *
 * Accumulation is fp32 with promotion once per 128-element k-block: the tensor core sums each k-block's 128 products on
 * its own (its internal precision inside a k-block is undocumented), and the kernel adds that partial into fp32
 * registers.  There is no fast-accumulation mode.  C is rounded once to OutT (round to nearest even; fp16 overflow
 * gives +-inf).  Scales are fp32 in device memory, read by the kernel only (a captured CUDA graph replays with the
 * values they hold at replay time):
 *   B200_SCALE_TENSOR  scale_a[0], scale_b[0]                         C = OutT((acc * scale_a[0]) * scale_b[0])
 *   B200_SCALE_ROW     scale_a[M], scale_b[N]                          C = OutT((acc[m,n] * scale_a[m]) * scale_b[n])
 *   B200_SCALE_BLOCK   scale_a [M, ceil(K/128)], M-major (element (m, kb) at m + kb * M, DeepGEMM's layout);
 *                      scale_b [ceil(N/128), ceil(K/128)], row-major (element (nb, kb) at nb * ceil(K/128) + kb).
 *                      Every k-block kb is promoted as acc = fma(partial, fp32(scale_a[m,kb] * scale_b[n/128,kb]), acc)
 *                      and C = OutT(acc) (DeepSeek-V3's 1 x 128 activation and 128 x 128 weight scales).
 * Constraints (B200_EINVAL, message naming the argument, before any CUDA call): a, b_nk, c, scale_a, scale_b not NULL;
 * a, b_nk, c 16-byte aligned, the scales 4-byte aligned; M, N, K >= 1; K % 16 == 0 (the TMA row stride); N % 8 == 0
 * (16-byte C stores); scale_recipe and c_dtype as above; c disjoint from a, b_nk and the scales.  Any M >= 1 and ragged
 * N and K are handled (k past K is zero-filled).  One launch, no workspace. */
#define B200_SCALE_TENSOR 0
#define B200_SCALE_ROW 1
#define B200_SCALE_BLOCK 2
int b200_gemm_e4m3(const void* a, const void* b_nk, void* c, const float* scale_a, const float* scale_b, int M, int N,
                   int K, int scale_recipe, int c_dtype, void* stream);

/* ------------------------------------------------------------------ merge_attn_states
 * Combine two partial attention results over disjoint key ranges (split-KV), SURVEY §8f-3.  Replaces
 *   merge_attn_states_cuda(output, output_lse?, prefix_output, prefix_lse, suffix_output, suffix_lse)
 *   (kernels/openai-triton/merge-attn-states/cuda_merge_attn_states.cu:19-95, 158-166).
 * output / prefix_output / suffix_output: [num_tokens, num_heads, head_size] of `dtype`, contiguous;
 * the lse tensors: [num_heads, num_tokens] fp32; output_lse may be NULL.  A +inf lse marks an empty
 * part and is treated as -inf, as in the reference.  A row whose two parts are both empty gets output 0
 * and output_lse -inf (never NaN), so it stays an empty part for the next merge.  head_size must be a
 * multiple of 16/sizeof(T).
 * Aliasing: output is either the same pointer as prefix_output / suffix_output (merging into an
 * accumulator in place) or disjoint from it; output_lse is disjoint from prefix_lse and suffix_lse.
 * Any other overlap returns B200_EINVAL.
 */
#define B200_DTYPE_F32 0
#define B200_DTYPE_F16 1
#define B200_DTYPE_BF16 2
#define B200_DTYPE_E4M3 3 /* OCP e4m3 (torch.float8_e4m3fn): KV caches of b200_kvcache_append_*; the e4m3 operands
                            * of b200_gemm_e4m3 have no dtype argument */
int b200_merge_attn_states(void* output, float* output_lse, const void* prefix_output,
                           const float* prefix_lse, const void* suffix_output, const float* suffix_lse,
                           int num_tokens, int num_heads, int head_size, int dtype, void* stream);

/* ------------------------------------------------------------------ rope / rms_norm (SURVEY §8f-4)
 * The element-wise steps either side of attention in the reference's catalogue.
 *
 * b200_rope_f32: rotary position embedding.  Replaces rope_f32 / rope_f32_v2 / rope_f32x4_pack(x, out)
 *   (kernels/rope/rope.cu:20-71, host :88-125).  x, out: [seq_len, hidden] fp32 contiguous; the pair
 *   (x[p,2i], x[p,2i+1]) is rotated by the angle p * theta^(-2i/hidden), theta = 10000.  hidden % 4 == 0.
 *
 * b200_rms_norm: y = x * rsqrt(mean(x^2, row) + 1e-5) * g.  Replaces rms_norm_f32{,x4}(x, y, g) and the
 *   seven rms_norm_f16* ops (kernels/rms-norm/rms_norm.cu:55-110, 161-415, host :493-771).  x, y:
 *   [rows, K] of `dtype` (B200_DTYPE_F32 or B200_DTYPE_F16), statistics always in fp32.  K must be a
 *   multiple of 16/sizeof(T) and at most 16384 (fp16) / 8192 (fp32).
 */
int b200_rope_f32(const float* x, float* out, int seq_len, int hidden, void* stream);

/* The same rotation on the attention operands: q, k fp16 [B,H,N,D] contiguous, the position of a row is its
 * sequence index n, pairs are (d = 2i, 2i+1), angle n * theta^(-2i/D); fp32 arithmetic, one rounding to fp16.
 * One launch rotates both tensors; each output is either its own input (q_out == q, k_out == k: in place) or
 * shares no byte with q, k or the other output, else B200_EINVAL.  q may be k when both outputs are separate
 * tensors; q == k in place is rejected (the two halves of the launch would rotate one buffer twice).  It is a pre-pass, not a fusion into the
 * attention main loop, on purpose: there K would be re-rotated once per query tile (N/256 times) with its
 * sin/cos on the MUFU pipe that already bounds the kernel; rotated once it costs one extra read + write of
 * q and k (HBM-bound).  D % 8 == 0. */
int b200_rope_qk_f16(const void* q, const void* k, void* q_out, void* k_out, int B, int H, int N, int D,
                     void* stream);
int b200_rms_norm(const void* x, void* y, float g, int rows, int K, int dtype, void* stream);

/* Attention with the RMS normalisation of every output row fused into the epilogue:
 *   o[b,h,i,:] = rms_norm(softmax(q_i K^T * scale) V) * rms_g     (eps 1e-5, statistics in fp32 over D)
 * i.e. b200_fmha_fwd_f16 followed by b200_rms_norm over rows of length D, without the round trip of O
 * through HBM (the row already sits in the registers of one thread when the epilogue runs).  rms_g <= 0
 * disables the normalisation (then identical to b200_fmha_fwd_f16_lse with an optional lse).  lse may be
 * NULL.  Supported for D <= 256 and for D = 384, 512 (there the two 256-column slabs of a query tile run as a
 * cluster of two CTAs and add up the row statistics through distributed shared memory); B200_ENOTSUP otherwise. */
int b200_fmha_fwd_f16_rmsnorm(const void* q, const void* k, const void* v, void* o, float* lse, int B,
                              int H, int N, int D, int v_transposed, float scale, float rms_g, void* stream);

/* Host-buffer convenience wrappers used for end-to-end timing: inputs are host
 * pointers (pinned or pageable); the call copies them to a cached device
 * workspace, runs the kernel and copies the result back, all on `stream`, and
 * returns after the stream has drained. */
int b200_hgemm_f16_host(const void* a, const void* b, void* c, int M, int N, int K, int b_layout,
                        void* stream);
int b200_fmha_fwd_f16_host(const void* q, const void* k, const void* v, void* o, int B, int H,
                           int N, int D, int v_transposed, float scale, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* LEETCUDA_B200_H_ */
