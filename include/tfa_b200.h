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

#ifdef __cplusplus
}
#endif
#endif /* TFA_B200_H_ */
