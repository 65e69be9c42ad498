/* tfa_b200.h -- C ABI of the H100-native (sm_90a) flash-attention forward.
 *
 * This is the drop-in boundary for the ONE hot path of 66RING/tiny-flash-attention:
 * the fused  O = softmax(scale * Q K^T [+ causal mask]) V  forward, plus the row
 * log-sum-exp.  Plain pointers and sizes only: no torch types cross this line.
 *
 * Reference interfaces replaced (paths relative to the reference project's root):
 *   - flash_attention_cutlass/include/attention_api.h:10-11 and
 *     flash_attention_cutlass/csrc/flash_attention.cu:741-772
 *       std::vector<torch::Tensor> flash_attention_v2_cutlass(q, k, v, is_causal, softmax_scale)
 *     -> tfa_fwd() (device pointers), wrapped 1:1 by the `attention_cutlass` extension
 *        (tiny-flash-attention_b200/csrc/attention_api.cpp).
 *   - flash_attention_cutlass/csrc/flash_attention.cu:731-739
 *       void run_flash_attn_cutlass(Flash_fwd_params&, cudaStream_t)   (POD params + stream)
 *     -> tfa_fwd_ex() (POD args incl. strides and the stream, which -- unlike the
 *        reference, flash_attention.cu:711 -- is honoured).
 *   - flash_attention_cutlass/csrc/flash.h:6-60  Qkv_params / Flash_fwd_params
 *     -> struct tfa_fwd_args.
 *
 * Error convention: every entry point returns 0 on success, a positive
 * cudaError_t on a CUDA failure, or a negative TFA_E* code on a bad argument.
 * Nothing ever calls exit() (the reference does: include/attention_api.cuh:20-29).
 * All launches are asynchronous on the caller's stream; no device-wide sync
 * (the reference does cudaDeviceSynchronize(): flash_attention.cu:768).
 */
#ifndef TFA_B200_H_
#define TFA_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TFA_ABI_VERSION 2   /* 2: + tfa_attn_* (grouped K/V heads, Sq != Sk, split-KV) */

/* dtype codes (reference: Qkv_params::is_bf16, flash.h:27) */
#define TFA_BF16 0
#define TFA_FP16 1
#define TFA_FP8_E4M3 2  /* input element type of the quantized calls only (tfa_kv_quant_args, tfa_qkv_quant_args) */

/* argument errors */
#define TFA_EINVAL_PTR    (-1)  /* null or not 16-byte aligned pointer           */
#define TFA_EINVAL_DIM    (-2)  /* head_dim not in {64, 128}                      */
#define TFA_EINVAL_SHAPE  (-3)  /* B, H or S < 1, or B*H > 65535*... overflow     */
#define TFA_EINVAL_DTYPE  (-4)  /* dtype not TFA_BF16 / TFA_FP16                  */
#define TFA_EINVAL_STRIDE (-5)  /* strides not expressible as a TMA tensor map    */
#define TFA_EDRIVER       (-6)  /* cuTensorMapEncodeTiled unavailable / failed    */
#define TFA_EARCH         (-7)  /* device is not compute capability 9.0           */
#define TFA_EDEVICE_FAULT (-8)  /* kernel watchdog fired; see tfa_debug_record()  */
#define TFA_EINVAL_SCALE  (-9)  /* softmax_scale negative, NaN or infinite         */
#define TFA_EINVAL_HEADS  (-10) /* Hq not a multiple of Hkv                         */
#define TFA_EINVAL_WORKSPACE (-11) /* split-KV asked for but workspace missing/small */
#define TFA_EINVAL_SEQLENS (-12)   /* cu_seqlens null / not 4-byte aligned, or max_seqlen_q not in [1, total_q] */
#define TFA_EINVAL_KVCACHE (-13)   /* KV cache: cache_seqlens / block_table null or misaligned, page size not a multiple
                                      of 128, num_blocks or max_blocks_per_seq < 1, one of k_new / v_new, Snew not in
                                      [1, capacity] */
#define TFA_EINVAL_ROTARY (-14)    /* rotary: cos / sin / q_rot null or misaligned, rotary_dim not an even multiple of 16
                                      in [16, D], seqlen_ro < capacity, or no k_new */
#define TFA_EINVAL_KVQUANT (-15)   /* FP8 cache: cache_dtype not TFA_FP8_E4M3, k_scale / v_scale not finite and > 0, or
                                      cache strides not multiples of 16 elements */
#define TFA_EINVAL_QKVQUANT (-16)  /* FP8 attention: qkv_dtype not TFA_FP8_E4M3, q_scale / k_scale / v_scale not finite and
                                      > 0, or q / k / v strides not multiples of 16 elements */

/* Extended argument block (POD), the analogue of Flash_fwd_params (flash.h:29-60).
 * Strides are in ELEMENTS.  The innermost (head_dim) stride must be 1.
 * Layout (B,H,S,D) contiguous == the reference's layout:
 *   stride_b = H*S*D, stride_h = S*D, stride_s = D.
 * Layout (B,S,H,D) (official flash_attn layout, test.py:71-75):
 *   stride_b = S*H*D, stride_h = D,   stride_s = H*D.
 * q, k, v and out all use the same strides (the reference also assumes this:
 * flash_attention.cu:409-424). lse is always (B,H,S) contiguous fp32, natural log:
 *   lse = scale*max + ln(sum)   (flash_attention.cu:623). */
typedef struct tfa_fwd_args {
  const void* q;
  const void* k;
  const void* v;
  void* out;            /* same dtype as q, or fp32 when out_fp32 != 0            */
  float* lse;           /* (B,H,S) fp32; may be NULL                              */
  int32_t B, H, S, D;
  int64_t stride_b, stride_h, stride_s;
  int32_t dtype;        /* TFA_BF16 / TFA_FP16                                    */
  int32_t is_causal;    /* top-left aligned causal mask (Sq == Sk)                */
  float softmax_scale;
  int32_t out_fp32;     /* debug/validation: skip the final 16-bit rounding       */
  void* stream;         /* cudaStream_t                                           */
} tfa_fwd_args;

int tfa_abi_version(void);

/* Device-pointer forward, (B,H,S,D) contiguous 16-bit tensors. */
int tfa_fwd(const void* q, const void* k, const void* v, void* out, float* lse,
            int B, int H, int S, int D, int dtype, int is_causal, float softmax_scale,
            void* cuda_stream);

/* Device-pointer forward with explicit strides / fp32 output / stream. */
int tfa_fwd_ex(const tfa_fwd_args* args);

/* Fused compute + exchange (SURVEY.md 8f row 1; the reference has no multi-GPU code, BASELINE.json's north_star
 * defines the exchange as an all-gather of O).  Same as tfa_fwd_ex(), and in the SAME kernel every 16-byte chunk
 * of O is additionally stored to `n_extra` (<= 7) other buffers with the same strides -- the peer GPUs' copies of
 * the gathered output, mapped into this process over NVLink (CUDA IPC / VMM / torch symmetric memory).  The stores
 * overlap the attention math tile by tile; the caller synchronises the ranks afterwards.  16-bit output only. */
int tfa_fwd_multi(const tfa_fwd_args* args, void* const* extra_out, int n_extra);

/* ---- generalised problem: grouped K/V heads (GQA/MQA), Sq != Sk, split-KV (SURVEY.md 8f rows 2-3) ----
 * Reference anchors: the CPU path takes k/v with their own sequence length and aligns the causal mask
 * bottom-right, kv_len = i + 1 + (Sk - Sq)  (flash_attention_c/csrc/attn.cpp:121-124,182-183); its archived
 * variant maps query head h to K/V head h / (Hq/Hkv)  (flash_attention_c/csrc/archive_)/attn.cpp:61,375); the
 * CuTe path carries the same fields dead (flash_attention_cutlass/csrc/flash.h:35-44) and emits the row LSE
 * "for backward" without a consumer (flash_attention.cu:353,615-623) -- split-KV is that consumer.
 *
 *   q, out : (B, Hq, Sq, D) through q_stride_* (elements, unit head_dim stride)
 *   k, v   : (B, Hkv, Sk, D) through kv_stride_*;  Hq % Hkv == 0
 *   lse    : (B, Hq, Sq) contiguous fp32, may be NULL
 *   causal : query row i sees keys j <= i + (Sk - Sq).  Rows that see no key (only when Sk < Sq) get
 *            out = 0 and lse = +inf (the CuTe epilogue's rule for an empty row, flash_attention.cu:620-623).
 *   num_splits: 1 = one pass.  n > 1 = the key range is cut into n chunks processed by independent CTAs (fills
 *            the GPU when B*Hq*ceil(Sq/128) is small), partial results go to `workspace`
 *            (tfa_attn_workspace_bytes()) and a second small kernel merges them through their LSEs.
 *            0 = let the library decide (splits only if a workspace large enough was passed).           */
typedef struct tfa_attn_args {
  const void* q;
  const void* k;
  const void* v;
  void* out;
  float* lse;
  int32_t B, Hq, Hkv, Sq, Sk, D;
  int64_t q_stride_b, q_stride_h, q_stride_s;
  int64_t kv_stride_b, kv_stride_h, kv_stride_s;
  int32_t dtype;
  int32_t is_causal;
  float softmax_scale;
  int32_t out_fp32;
  int32_t num_splits;
  void* workspace;          /* device memory, 16-byte aligned; may be NULL when num_splits <= 1 */
  size_t workspace_bytes;
  void* stream;
} tfa_attn_args;

int tfa_attn_fwd(const tfa_attn_args* args);
/* The split count tfa_attn_fwd() would use for args->num_splits (resolves 0 = auto, clamps n), >= 1. */
int tfa_attn_num_splits(const tfa_attn_args* args);
/* Workspace needed for `num_splits` (as returned above): num_splits * B*Hq*Sq * (D + 1) * 4 bytes; 0 for 1. */
size_t tfa_attn_workspace_bytes(const tfa_attn_args* args, int num_splits);

/* ---- variable-length batch (packed sequences, the flash-attn "varlen" interface) ----
 * Added without an ABI version change (TFA_ABI_VERSION stays 2): callers detect it by the exported symbol
 * tfa_attn_varlen_fwd.
 *
 *   q        : (total_q, Hq, D) through q_stride_s / q_stride_h (elements, unit head_dim stride)
 *   k, v     : (total_k, Hkv, D) through kv_stride_s / kv_stride_h;  Hq % Hkv == 0.  The strides let q, k and v
 *              be views of one packed (total, 3, H, D) tensor.
 *   out      : (total_q, Hq, D) contiguous, dtype of q, or fp32 when out_fp32 != 0
 *   lse      : (Hq, total_q) contiguous fp32, natural log; may be NULL
 *   cu_seqlens_q, cu_seqlens_k : int32 DEVICE arrays of B + 1 entries, cu[0] = 0, non-decreasing, cu[B] = total.
 *              Sequence b is rows [cu_q[b], cu_q[b+1]) of q/out and rows [cu_k[b], cu_k[b+1]) of k/v, and is the
 *              problem tfa_attn_fwd() solves: query head h reads K/V head h / (Hq/Hkv); causal is bottom-right
 *              aligned, row i sees keys j <= i + (Sk_b - Sq_b).  Rows that see no key (causal Sq_b > Sk_b, or
 *              Sk_b == 0) get out = 0 and lse = +inf; a sequence with Sq_b == 0 writes nothing.
 *   total_q, total_k : >= 1.
 *   max_seqlen_q : >= every Sq_b, in [1, total_q].  The host never reads cu_seqlens: the kernel does, clamping
 *              every entry to [0, total], so malformed contents cannot make it write outside out and lse.  Rows of
 *              a sequence beyond its first max_seqlen_q are not computed and keep what out / lse held (as in
 *              flash-attn).
 * One kernel launch per call, nothing read back to the host: the call can be captured in a CUDA graph and replayed
 * with new cu_seqlens contents of the same totals.  No split-KV. */
typedef struct tfa_attn_varlen_args {
  const void* q;
  const void* k;
  const void* v;
  void* out;
  float* lse;
  const int32_t* cu_seqlens_q;
  const int32_t* cu_seqlens_k;
  int32_t B, Hq, Hkv, D;
  int32_t total_q, total_k, max_seqlen_q;
  int64_t q_stride_s, q_stride_h;
  int64_t kv_stride_s, kv_stride_h;
  int32_t dtype;
  int32_t is_causal;
  float softmax_scale;
  int32_t out_fp32;
  void* stream;
} tfa_attn_varlen_args;

int tfa_attn_varlen_fwd(const tfa_attn_varlen_args* args);

/* ---- attention against a (paged) KV cache: the decode step of a serving loop (flash-attn's flash_attn_with_kvcache;
 * with rotary see tfa_attn_kvcache_rotary_fwd below) ----
 * Added without an ABI version change (TFA_ABI_VERSION stays 2): callers detect it by the exported symbol
 * tfa_attn_kvcache_fwd.
 *
 *   q, out   : (B, Sq, Hq, D) through q_stride_* (elements, unit head_dim stride); out uses q's strides and is q's
 *              dtype, or fp32 when out_fp32 != 0.  Sq >= 1: 1 for decode, a few for speculative verification.
 *   lse      : (B, Hq, Sq) contiguous fp32, natural log; may be NULL
 *   k_cache, v_cache : (num_blocks, page_block_size, Hkv, D) through cache_stride_* (block, row, head), shared by both;
 *              Hq % Hkv == 0.
 *   block_table : int32 DEVICE array (B, max_blocks_per_seq) with row stride block_table_stride: logical page p of
 *              sequence b is physical block block_table[b * stride + p].  page_block_size must be a multiple of 128.
 *              NULL: a contiguous cache (B, capacity, Hkv, D) -- pass num_blocks = B, max_blocks_per_seq = 1 and
 *              page_block_size = capacity (any value >= 1).
 *   cache_seqlens : int32 DEVICE array (B): keys already cached per sequence.
 *   k_new, v_new : optional (B, Snew, Hkv, D) through new_stride_* (both or neither).  They are written into the cache
 *              at keys [L_b, L_b + Snew) before the attention, in place; cache_seqlens is not incremented.
 *   capacity = max_blocks_per_seq * page_block_size;  L_b = clamp(cache_seqlens[b], 0, capacity - Snew) (Snew = 0
 *              without k_new).  Sequence b attends to its first K_b = L_b + Snew keys: query head h reads K/V head
 *              h / (Hq/Hkv), causal is bottom-right aligned (row i sees keys j <= i + K_b - Sq), rows that see no key
 *              get out = 0 and lse = +inf.  Cache slots past K_b may hold anything (NaN included) and do not change the
 *              result.
 *   num_splits, workspace : as tfa_attn_args.  tfa_attn_num_splits() / tfa_attn_workspace_bytes() on the dense
 *              problem (B, Hq, Sq, Sk = capacity) give the split count and the workspace it needs.
 * The host never reads cache_seqlens or block_table: the call (append included) can be captured in a CUDA graph and
 * replayed with new contents.  The kernels clamp the lengths; a block-table entry outside [0, num_blocks) is never
 * written through (the append drops that token) and reads through it return zeros, so malformed contents cannot make
 * a store leave out, lse or the cache.  Launches: 1, + 1 with k_new, + 1 with split-KV. */
typedef struct tfa_attn_kvcache_args {
  const void* q;
  void* k_cache;
  void* v_cache;
  const void* k_new;        /* may be NULL (then v_new must be NULL too) */
  const void* v_new;
  void* out;
  float* lse;
  const int32_t* cache_seqlens;
  const int32_t* block_table;  /* may be NULL: contiguous cache */
  int32_t B, Hq, Hkv, Sq, D;
  int32_t num_blocks, page_block_size, max_blocks_per_seq;
  int32_t Snew;             /* rows of k_new / v_new; ignored without them */
  int64_t q_stride_b, q_stride_s, q_stride_h;
  int64_t cache_stride_block, cache_stride_s, cache_stride_h;
  int64_t block_table_stride;
  int64_t new_stride_b, new_stride_s, new_stride_h;
  int32_t dtype;
  int32_t is_causal;
  float softmax_scale;
  int32_t out_fp32;
  int32_t num_splits;
  void* workspace;
  size_t workspace_bytes;
  void* stream;
} tfa_attn_kvcache_args;

int tfa_attn_kvcache_fwd(const tfa_attn_kvcache_args* args);

/* ---- the KV-cache forward with rotary position embedding (flash-attn's flash_attn_with_kvcache with rotary_cos,
 * rotary_sin and rotary_interleaved) ----
 * Added without an ABI version change (TFA_ABI_VERSION stays 2): callers detect it by the exported symbol
 * tfa_attn_kvcache_rotary_fwd.  tfa_attn_kvcache_fwd() with, before the attention, q and k_new rotated at their
 * absolute positions in one launch: rot(q) goes to q_rot, which the attention reads in place of q, and rot(k_new) with
 * the unrotated v_new goes into the cache.  The caller's q and k_new are not modified.
 *
 *   cos, sin   : (seqlen_ro, rotary_dim / 2) contiguous DEVICE arrays in q's dtype, 16-byte aligned.
 *   seqlen_ro  : >= capacity (= max_blocks_per_seq * page_block_size).
 *   rotary_dim : a multiple of 16 in [16, D].  Dimensions [rotary_dim, D) pass through unchanged.
 *   interleaved: 0 = GPT-NeoX pairs (j, j + rotary_dim/2), != 0 = GPT-J pairs (2j, 2j+1); pair j takes cos[pos][j] and
 *              sin[pos][j], and becomes x0' = x0 c - x1 s, x1' = x0 s + x1 c, computed in fp32 with one rounding per
 *              operation (no FMA) and rounded once to q's dtype.
 *   q_rot      : (B, Sq, Hq, D) contiguous DEVICE scratch in q's dtype, 16-byte aligned; it must not overlap any other
 *              argument.  Holds rot(q) after the call.
 *   positions  : with L_b the clamped cached length of tfa_attn_kvcache_fwd(), appended key i of sequence b is rotated
 *              at L_b + i; query row i at L_b + i when causal, at L_b for every row otherwise (equal to the key
 *              positions when Sq == Snew).  A query position past seqlen_ro - 1 (Sq > Snew near the capacity) is
 *              clamped to seqlen_ro - 1.
 * k_new / v_new are required (TFA_EINVAL_ROTARY otherwise).  out keeps q's strides.  Every argument is checked before
 * any device work.  Launches: 2 (the rotary append, the attention), + 1 with split-KV; CUDA-graph capturable as
 * tfa_attn_kvcache_fwd(). */
typedef struct tfa_rotary_args {
  const void* cos;
  const void* sin;
  int32_t seqlen_ro, rotary_dim, interleaved;
  void* q_rot;
} tfa_rotary_args;

int tfa_attn_kvcache_rotary_fwd(const tfa_attn_kvcache_args* args, const tfa_rotary_args* rotary);

/* ---- a variable-length batch of queries against a (paged) KV cache: the mixed prefill / decode step of a
 * continuous-batching loop (flash-attn's flash_attn_varlen_func with block_table and seqused_k) ----
 * Added without an ABI version change (TFA_ABI_VERSION stays 2): callers detect it by the exported symbol
 * tfa_attn_varlen_kvcache_fwd.  Queries as tfa_attn_varlen_fwd(), keys and values as tfa_attn_kvcache_fwd().
 *
 *   q        : (total_q, Hq, D) through q_stride_s / q_stride_h (elements, unit head_dim stride)
 *   out      : (total_q, Hq, D) contiguous, dtype of q, or fp32 when out_fp32 != 0
 *   lse      : (Hq, total_q) contiguous fp32, natural log; may be NULL
 *   cu_seqlens_q : int32 DEVICE array of B + 1 offsets: sequence b is rows [cu[b], cu[b+1]) of q / out.  Its query
 *              count Sq_b is taken with the offsets clamped to [0, total_q]; n_b = min(Sq_b, max_seqlen_q).
 *   max_seqlen_q : in [1, total_q], >= every Sq_b.  Rows of a sequence beyond its first max_seqlen_q are neither
 *              computed nor appended and keep what out / lse held; the sequence is then its first n_b rows.
 *   k_cache, v_cache, block_table, num_blocks, page_block_size, max_blocks_per_seq, cache_stride_*,
 *   block_table_stride, cache_seqlens : as tfa_attn_kvcache_args (page_block_size % 128 == 0 with a table; NULL
 *              table: a contiguous (B, capacity, Hkv, D) cache).  capacity = max_blocks_per_seq * page_block_size.
 *   k_new, v_new : optional (both or neither), packed (total_q, Hkv, D) through new_stride_s / new_stride_h, sharing
 *              cu_seqlens_q with q: row cu[b] + i is key L_b + i of sequence b.  Written into the cache in place
 *              before the attention; cache_seqlens is not incremented.
 *   lengths  : with k_new, L_b = clamp(cache_seqlens[b], 0, max(capacity - n_b, 0)) and K_b = min(L_b + n_b,
 *              capacity); an appended token past the capacity or whose block-table entry lies outside
 *              [0, num_blocks) is dropped.  Without k_new (the caller wrote the step's keys: seqused_k),
 *              K_b = clamp(cache_seqlens[b], 0, capacity).
 *   attention: sequence b's n_b rows attend to its first K_b keys.  Query head h reads K/V head h / (Hq/Hkv); causal
 *              is bottom-right aligned, row i sees keys j <= i + K_b - n_b; rows that see no key get out = 0 and
 *              lse = +inf; a sequence with Sq_b == 0 writes nothing.  Cache slots past K_b may hold anything (NaN
 *              included) and do not change the result.
 * The host never reads cu_seqlens_q, cache_seqlens or block_table: the call (append included) can be captured in a
 * CUDA graph and replayed with new contents of the same total_q.  The kernels clamp every length and offset, so
 * malformed contents cannot make a store leave out, lse or a sequence's appended cache slots.  No split-KV (a
 * decode-only batch keeps tfa_attn_kvcache_fwd(), which has it).  Every argument is checked before any device work.
 * Launches: 1, + 1 with k_new. */
typedef struct tfa_attn_varlen_kvcache_args {
  const void* q;
  void* k_cache;
  void* v_cache;
  const void* k_new;        /* may be NULL (then v_new must be NULL too) */
  const void* v_new;
  void* out;
  float* lse;
  const int32_t* cu_seqlens_q;
  const int32_t* cache_seqlens;
  const int32_t* block_table;  /* may be NULL: contiguous cache */
  int32_t B, Hq, Hkv, D;
  int32_t total_q, max_seqlen_q;
  int32_t num_blocks, page_block_size, max_blocks_per_seq;
  int64_t q_stride_s, q_stride_h;
  int64_t cache_stride_block, cache_stride_s, cache_stride_h;
  int64_t block_table_stride;
  int64_t new_stride_s, new_stride_h;
  int32_t dtype;
  int32_t is_causal;
  float softmax_scale;
  int32_t out_fp32;
  void* stream;
} tfa_attn_varlen_kvcache_args;

int tfa_attn_varlen_kvcache_fwd(const tfa_attn_varlen_kvcache_args* args);

/* ---- the KV-cache calls against an FP8 (e4m3) cache with per-tensor scales (vLLM's kv_cache_dtype="fp8") ----
 * Added without an ABI version change (TFA_ABI_VERSION stays 2): callers detect them by the exported symbols
 * tfa_attn_kvcache_fp8_fwd and tfa_attn_varlen_kvcache_fp8_fwd.  tfa_attn_kvcache_fwd() (with `rotary`:
 * tfa_attn_kvcache_rotary_fwd()) and tfa_attn_varlen_kvcache_fwd() with k_cache / v_cache holding one byte per element.
 * args->dtype stays q's dtype; q, k_new, v_new, out and lse keep their types.  Cache strides are in elements (bytes)
 * and must be multiples of 16.
 *
 *   cache values : an element x8 (e4m3 codes, torch.float8_e4m3fn) stands for k_scale * x8 in K, v_scale * x8 in V.
 *   append       : key K8 = e4m3_rn_satfinite(k_new / k_scale), value V8 = e4m3_rn_satfinite(v_new / v_scale): IEEE
 *                  fp32 division, round to nearest-even, saturated to +-448 -- bit-identical to torch's
 *                  (x.float() / scale).clamp(-448, 448).to(torch.float8_e4m3fn).  With rotary the rotated key is rounded
 *                  to q's dtype as tfa_attn_kvcache_rotary_fwd() stores it, then quantized.  Lengths, the table,
 *                  dropped tokens and the capacity clamp are those of the 16-bit calls.
 *   attention    : every finite e4m3 code widens exactly to bf16 / fp16; the kernel runs the 16-bit call's arithmetic
 *                  on the widened cache with softmax scale s' = fp32(softmax_scale * k_scale) and the output scaled by
 *                  v_scale.  So for v_scale a power of two, out and lse are bit-identical to the 16-bit call on
 *                  k8.to(q dtype) / v8.to(q dtype) with softmax_scale = s', its out multiplied by v_scale; for other
 *                  v_scale they differ by the rounding of that product.  Slots past K_b may hold any byte, NaN codes
 *                  0x7f / 0xff included, and do not change the result.
 * s' must stay a normal fp32 number: when it overflows, or when softmax_scale > 0 and it underflows below FLT_MIN (which
 * would make the attention uniform), the call returns TFA_EINVAL_SCALE.
 * Every check runs before any device work, those of the 16-bit call first (TFA_EINVAL_KVQUANT after them).  Launches
 * and CUDA-graph capture as the 16-bit calls; split-KV as tfa_attn_kvcache_fwd() (the varlen call has none). */
typedef struct tfa_kv_quant_args {
  int32_t cache_dtype;      /* TFA_FP8_E4M3 */
  float k_scale, v_scale;   /* finite, > 0 */
} tfa_kv_quant_args;

int tfa_attn_kvcache_fp8_fwd(const tfa_attn_kvcache_args* args, const tfa_rotary_args* rotary /* NULL: none */,
                             const tfa_kv_quant_args* quant);
int tfa_attn_varlen_kvcache_fp8_fwd(const tfa_attn_varlen_kvcache_args* args, const tfa_kv_quant_args* quant);

/* ---- attention on FP8 (e4m3) q, k and v with per-tensor scales, both products on FP8 tensor cores (FlashAttention-3's
 * descale_q / descale_k / descale_v) ----
 * Added without an ABI version change (TFA_ABI_VERSION stays 2): callers detect it by the exported symbol
 * tfa_attn_fp8_fwd.  The problem of tfa_attn_fwd(), unchanged -- grouped K/V heads, Sq != Sk with the bottom-right
 * causal mask, key-less rows out = 0 / lse = +inf, split-KV through num_splits / workspace (tfa_attn_num_splits() and
 * tfa_attn_workspace_bytes() on the same args), out_fp32 -- with q, k and v holding one byte per element.
 *
 *   q, k, v  : e4m3 codes (torch.float8_e4m3fn).  Strides are in elements, so in bytes, and must be multiples of 16.
 *   dtype    : the OUTPUT dtype, TFA_BF16 or TFA_FP16 (or fp32 with out_fp32).  out uses q's element strides; lse is
 *              fp32 (B, Hq, Sq) as everywhere.
 *   scales   : a code x8 stands for q_scale * x8 in Q, k_scale * x8 in K, v_scale * x8 in V; out and lse are those of
 *              the dequantized problem.  The kernel computes S = Q8 K8^T on e4m3 wgmma with fp32 accumulation, takes the
 *              softmax with scale s' = fp32(fp32(softmax_scale * q_scale) * k_scale) (that order), rounds P to e4m3
 *              (round to nearest even; P <= 2^8), computes P8 V8 on e4m3 wgmma and multiplies O by v_scale.
 * s' must stay a normal fp32 number: when it overflows, or when softmax_scale > 0 and it underflows below FLT_MIN, the
 * call returns TFA_EINVAL_SCALE.  Every check runs before any device work, those of tfa_attn_fwd() first, in its order,
 * then TFA_EINVAL_QKVQUANT, then TFA_EINVAL_SCALE for s'.  Launches: 1, + 1 with split-KV.  Callers quantize, e.g.
 * (x / s).clamp(-448, 448).to(torch.float8_e4m3fn). */
typedef struct tfa_qkv_quant_args {
  int32_t qkv_dtype;                 /* TFA_FP8_E4M3 */
  float q_scale, k_scale, v_scale;   /* finite, > 0 */
} tfa_qkv_quant_args;

int tfa_attn_fp8_fwd(const tfa_attn_args* args, const tfa_qkv_quant_args* quant);

/* ---- the variable-length batch on FP8 (e4m3) q, k and v with per-tensor scales (FlashAttention-3's
 * flash_attn_varlen_func with descale_q / descale_k / descale_v) ----
 * Added without an ABI version change (TFA_ABI_VERSION stays 2): callers detect it by the exported symbol
 * tfa_attn_varlen_fp8_fwd.  The problem of tfa_attn_varlen_fwd(), unchanged -- packed q (total_q, Hq, D) and k / v
 * (total_k, Hkv, D), cu_seqlens_q / cu_seqlens_k read on the device only, grouped K/V heads, the bottom-right causal
 * mask per sequence, key-less rows out = 0 / lse = +inf, rows beyond max_seqlen_q untouched, out_fp32, no split-KV --
 * with q, k and v holding one byte per element, and the arithmetic and scales of tfa_attn_fp8_fwd().
 *
 *   q, k, v  : e4m3 codes (torch.float8_e4m3fn).  Strides are in elements, so in bytes, and must be multiples of 16.
 *   dtype    : the OUTPUT dtype, TFA_BF16 or TFA_FP16 (or fp32 with out_fp32).  out is (total_q, Hq, D) contiguous;
 *              lse is fp32 (Hq, total_q) as for tfa_attn_varlen_fwd().
 *   scales   : as tfa_attn_fp8_fwd(): s' = fp32(fp32(softmax_scale * q_scale) * k_scale), P rounded to e4m3, O multiplied
 *              by v_scale.  Each sequence's out and lse are bit-identical to tfa_attn_fp8_fwd() (num_splits = 1) on that
 *              sequence alone; the keys of the neighbouring sequences may hold any byte, NaN codes 0x7f / 0xff included,
 *              and do not change the result.
 * Every check runs before any device work: those of tfa_attn_varlen_fwd() first, in its order, then
 * TFA_EINVAL_QKVQUANT, then TFA_EINVAL_SCALE for s'.  Launches: 1.  Nothing is read back to the host: the call can be
 * captured in a CUDA graph and replayed with new cu_seqlens contents of the same totals. */
int tfa_attn_varlen_fp8_fwd(const tfa_attn_varlen_args* args, const tfa_qkv_quant_args* quant);

/* Host-buffer forward: q/k/v/out/lse are HOST pointers ((B,H,S,D) contiguous; pinned
 * memory gives full PCIe speed).  Copies in, runs tfa_fwd per (batch*head) chunk on
 * `n_streams` internal streams so H2D, compute and D2H overlap, copies out, and
 * returns after everything completed.  Workspace is cached between calls;
 * tfa_host_release() frees it. */
int tfa_fwd_host(const void* q, const void* k, const void* v, void* out, float* lse,
                 int B, int H, int S, int D, int dtype, int is_causal, float softmax_scale,
                 int n_chunks);
void tfa_host_release(void);

/* Number of kernels this library has launched since load (bench.py's gpu_launches). */
unsigned long long tfa_launch_count(void);

/* Watchdog record of the last device fault: 8 words
 * {flag, block, thread, site, iter, parity, aux0, aux1}; flag == 0 means clean. */
int tfa_debug_record(unsigned int out[8]);
void tfa_debug_clear(void);

const char* tfa_error_string(int code);

/* ---- bring-up self tests (device side of tests/test_umma_primitives.py) ----
 * Each runs one tiny kernel exercising one primitive the forward is built from and
 * writes raw results for the host to check.  All pointers are device pointers.   */

/* TMA 3-D tiled load, SWIZZLE_128B: copies the (64 x 128) box at (x0, y0, z0) of a
 * (D, S, BH) 16-bit tensor into shared memory and dumps the 16 KB verbatim.       */
int tfa_selftest_tma(const void* src, int D, int S, int BH, int x0, int y0, int z0,
                     void* dump_16k, void* stream);

/* One wgmma chain: C(128 x N, fp32) = A(128 x K) * B, operands staged by TMA, two m64 halves.
 *   mode 0: SS, B is (N x K) K-major       (the Q K^T contraction)
 *   mode 1: SS, B is (K x N) MN-major      (V consumed in place)
 *   mode 2: RS, A in registers (16-bit pairs), B (K x N) MN-major  (the P V contraction)
 * K in {64,128}, N in {64,128}.  `knobs` (may be NULL) overrides descriptor fields:
 *   knobs[0] = LBO bytes (0 = default), knobs[1] = SBO bytes (0 = default),
 *   knobs[2] = k-step byte advance (0 = default), knobs[3] = flags
 *              (bit0: swap packing order of the two 16-bit halves of register A). */
int tfa_selftest_umma(const void* a, const void* b, float* c, int N, int K, int mode,
                      int dtype, const int* knobs, void* stream);

/* e4m3 wgmma chains with fp32 accumulation, C(128 x N) += chain x A(128 x K) * B, two m64 halves, K in {64, 128}: the
 * accumulator starts at c's contents and takes the K-deep chain `chain` times (1..4096), chain x K / 32 k-steps.
 *   mode 0: SS, A (128 x K) and B (N x K) both K-major e4m3, staged by TMA with the 128-byte (K = 128) or 64-byte
 *           (K = 64) swizzle; N = 128 (the Q K^T contraction).
 *   mode 1: RS, A (128 x 128 keys) in registers, packed from the fp32 accumulator layout in fp8_p_key order, and B
 *           (N x 128 keys) K-major in shared memory with its keys in the same order, written by the V^T converter from
 *           the (128 keys x N) row-major b; N in {64, 128} (the P V contraction).  K must be 128.
 * a, b hold e4m3 codes (row-major as described), c fp32 (128 x N), read and overwritten. */
int tfa_selftest_wgmma_fp8(const void* a, const void* b, float* c, int N, int K, int mode, int chain, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* TFA_B200_H_ */
