// fa_fwd_sm90.cuh -- the fused attention-forward kernel for sm_90a (H100).
//
//   O = softmax(scale * Q K^T  [+ causal mask]) V ,  LSE = scale*max + ln(sum)
//
// One hand-written kernel replaces the reference's CuTe/sm80 kernel (flash_attention_cutlass/csrc/
// flash_attention.cu:373-685 of the reference).  The algorithm is the same FA-2 recurrence (SURVEY.md A.1); the
// machine mapping is Hopper's:
//
//   * one work item = TWO 64-row Q tiles of one (batch, head) that share every K/V tile (reference: one 64-row tile
//     per CTA, flash_attention.cu:695-699); items are taken in chunks of 8 heads, heaviest causal pair first across the
//     chunk (decode_work), so K/V stay L2 resident and the grid's tail is light;
//   * Q/K/V tiles are staged HBM -> shared memory by TMA (SWIZZLE_128B boxes of 64 x 128 elements) behind mbarriers,
//     a 4 (D=128) or 8 (D=64) deep K/V ring filled by one producer warp (reference: cp.async, single buffered,
//     flash_attention.cu:521-525,556-565,581-590);
//   * S = Q K^T and O += P V run on wgmma with fp32 accumulators in registers: S is an SS-form wgmma (Q and K both
//     K-major in shared memory), O is an RS-form wgmma whose A operand P is the softmax warpgroup's own registers and
//     whose B operand is the V tile consumed in place as an MN-major operand -- no transpose, no ldmatrix.trans
//     (reference: mma.sync m16n8k16 + ldmatrix(.trans), flash_attention.cu:84-132, kernel_traits.h:26-39);
//   * inside a warpgroup, S_{j+1} = Q K_{j+1}^T and O += P_j V_j are issued together, so the tensor cores work on both
//     while the warpgroup's softmax of S_{j+1} waits only for the first; the two warpgroups interleave on their own;
//   * softmax: each thread holds two rows' quarter (32 columns each), row max / row sum over the 4-thread quad; exp is
//     ex2.approx with scale*log2(e) folded into one FFMA; O is rescaled lazily, only when the running max moved by more
//     than 2^8 (reference: unconditional rescale every tile, flash_attention.cu:264-316);
//   * causal: KV tiles above the diagonal are skipped, only tiles crossing it are masked
//     (reference: flash_attention.cu:536-540,576-578 with 64-wide tiles);
//   * epilogue: O/l -> 16-bit -> swizzled shared-memory staging -> coalesced 128-bit st.global.v4
//     (reference: flash_attention.cu:608-663), optionally repeated for up to 7 peer GPUs' buffers (fused
//     all-gather, tfa_fwd_multi); LSE by the row-owner threads (:666-683).
//
// Warp roles (384 threads): warpgroup 0 is the producer (one lane of warp 0 issues every TMA load; the warpgroup
// gives its registers to the others), warpgroups 1 and 2 run Q tile 0 and 1: wgmma, softmax, epilogue.
// PERSIST = false: one CTA per work item.  PERSIST = true: one CTA per SM walks the items blockIdx.x, +gridDim.x, ...
// and its producer runs ahead into the next item's Q and K/V while the softmax warpgroups finish the current one.
// MODE (the problem the grid solves): kDense = (B, H, S, D) tensors; kVarlen = a packed variable-length batch, each
// item reads its sequence's offsets and lengths from cu_seqlens; kCache = decode against a (paged) KV cache, each item
// reads its sequence's cached length from cache_seqlens and its K/V boxes' pages from a block table; kVarlenCache =
// both at once, a packed variable-length batch of queries (cu_seqlens) against a (paged) KV cache.  kCacheFp8 and
// kVarlenCacheFp8 are kCache and kVarlenCache against an FP8 (e4m3) cache: the TMA lane loads raw e4m3 tiles into a
// ring of their own, and producer warps 1-3 (the converter) widen each into the 16-bit K/V ring slot the softmax
// warpgroups read, exactly, in the layout TMA gives a 16-bit tile; their code does not change.  kDenseFp8 and
// kVarlenFp8 are kDense and kVarlen with Q, K and V in e4m3 and both products on 8-bit wgmma (qkv8_mode()).
#pragma once
#include "ptx_sm90.cuh"

namespace tfa {

enum : int {
  kDense = 0, kVarlen = 1, kCache = 2, kVarlenCache = 3, kCacheFp8 = 4, kVarlenCacheFp8 = 5, kDenseFp8 = 6, kVarlenFp8 = 7
};
// The problem an FP8-cache mode solves is that of its 16-bit mode: they differ only in how K/V reach the ring.
__host__ __device__ constexpr bool fp8_mode(int mode) { return mode == kCacheFp8 || mode == kVarlenCacheFp8; }
// kDenseFp8 / kVarlenFp8 solve the dense / varlen problem with Q, K and V in e4m3 and both products on 8-bit wgmma
// (fp8_mode() is false for them: that predicate means "widen K/V to 16 bits").
__host__ __device__ constexpr bool qkv8_mode(int mode) { return mode == kDenseFp8 || mode == kVarlenFp8; }
__host__ __device__ constexpr int base_mode(int mode) {
  return mode == kCacheFp8 ? kCache : mode == kVarlenCacheFp8 ? kVarlenCache : mode == kDenseFp8 ? kDense
       : mode == kVarlenFp8 ? kVarlen : mode;
}

// ---- kDenseFp8: P as the 8-bit A operand without shuffles ----
// The fp32 accumulator gives thread (g, tq) keys 8i + 2tq, +1 of rows g and g + 8; the 8-bit A fragment wants of it
// columns 4tq .. 4tq + 3 (and 16 + those) of each 32-key k-step.  So A column c of a 32-key block holds key
// pi(c) = 8 (x >> 1) + 2 tq + (x & 1) for c = 4 tq + x < 16, and pi(16 + c) = 16 + pi(c): every thread packs only its
// own values, and the converter writes V^T's keys in the same order.  The sum over keys does not depend on it.
__host__ __device__ constexpr int fp8_p_key(int c) {
  return (c & 16) + 8 * ((c >> 1) & 1) + 2 * ((c >> 2) & 3) + (c & 1);
}
// The packer: byte x of A register r (0..3) of a k-step is accumulator element s[16 kk + fp8_pack_src(r, x)] (the
// fp32 layout: s[4 i + 2 h + e] = row g + 8 h, key 8 i + 2 tq + e).  Derived from pi at tq = 0: 2 tq only shifts keys.
__host__ __device__ constexpr int fp8_pack_src(int r, int x) {
  return 4 * (fp8_p_key(16 * (r >> 1) + x) >> 3) + 2 * (r & 1) + (fp8_p_key(16 * (r >> 1) + x) & 1);
}
// The converter: position p (0..127) of a V^T row holds key fp8_vt_key(p) of the 128-key tile.
__host__ __device__ constexpr int fp8_vt_key(int p) { return (p & ~31) + fp8_p_key(p & 31); }

// ---- KV-cache address math, host-callable so that a CPU test can check it exhaustively (tests/test_kvcache.py) ----
// Keys attended by sequence b: its cached length clamped to [0, capacity - snew], plus the snew appended keys.  The
// clamp keeps every append inside the sequence's capacity whatever cache_seqlens holds.
__host__ __device__ __forceinline__ int cache_len(int raw, int capacity, int snew) {
  return min(max(raw, 0), capacity - snew);
}
// Logical key `key` (0 <= key < capacity) of sequence b -> (physical block, row inside it).  Without a block table
// the cache is contiguous, one page of `page` = capacity rows per sequence, and the block is b.  The entry is
// returned as stored: the TMA loads bounds-check it in hardware, the append checks it with block_ok().
__host__ __device__ __forceinline__ void page_lookup(const int* block_table, long long bt_stride, int b, int key,
                                                     int page, int& blk, int& row) {
  const int pg = key / page;
  blk = block_table ? block_table[b * bt_stride + pg] : b;
  row = key - pg * page;
}
__host__ __device__ __forceinline__ bool block_ok(int blk, int num_blocks) { return blk >= 0 && blk < num_blocks; }
// Sequence b appends n keys (n = 0: no append) and keeps the first min(n, capacity) of them: the rest do not fit and
// are dropped.  n exceeds the capacity only in the variable-length call, whose n_b = min(Sq_b, max_seqlen_q) the host
// does not know.  L = its clamped cached length (cache_len of the kept count), K = the keys it attends.
__host__ __device__ __forceinline__ void cache_lens(int raw, int capacity, int n, int& L, int& K) {
  const int kept = min(n, capacity);
  L = cache_len(raw, capacity, kept);
  K = L + kept;
}
// Element offset, in a cache with (block, row, head) element strides cs_b / cs_s / cs_h, of appended token i
// (0 <= i < n) of sequence b at head h (raw = cache_seqlens[b]), or -1 when the token is dropped: it does not fit the
// capacity (i >= min(n, capacity)) or its block-table entry lies outside [0, num_blocks).
__host__ __device__ __forceinline__ long long append_offset(int raw, const int* block_table, long long bt_stride, int b,
                                                            int i, int h, int page, int capacity, int n, int num_blocks,
                                                            long long cs_b, long long cs_s, long long cs_h) {
  int L, K;
  cache_lens(raw, capacity, n, L, K);
  const int key = L + i;
  if (key >= K) return -1;
  int blk, row;
  page_lookup(block_table, bt_stride, b, key, page, blk, row);
  if (!block_ok(blk, num_blocks)) return -1;
  return blk * cs_b + row * cs_s + h * cs_h;
}

// Where a call's results go: row `row` of (batch b, head h) has its O at element b*sb + h*sh + row*ss of out and its
// LSE at element b*lse_sb + h*lse_sh + row of lse.  The host builds it once per call (tfa_api.cu); the forward and the
// combine address out / lse through it.  Packed (varlen) layouts have sb = lse_sb = 0 and count `row` from the packed
// tensors' first row.
struct OutLayout {
  long long sb, sh, ss;
  long long lse_sb, lse_sh;
  __host__ __device__ __forceinline__ long long o(long long b, long long h, long long row) const {
    return b * sb + h * sh + row * ss;
  }
  __host__ __device__ __forceinline__ long long lse(long long b, long long h, long long row) const {
    return b * lse_sb + h * lse_sh + row;
  }
};

struct FwdParams {
  void* out;          // 16-bit output at `ol`
  // Fused exchange (multi-GPU): when n_extra_dst > 0 every 16-byte chunk of O is ALSO stored to these buffers
  // (same layout) -- peer GPUs' copies of the gathered output, mapped over NVLink.  Replaces the all-gather.
  void* extra_dst[7];
  int n_extra_dst;
  float* out_f32;     // fp32 output (validation build, or the split-KV partials), at `ol`
  float* lse;         // fp32 at `ol`, or nullptr
  OutLayout ol;       // the caller's layout, or that of one split's partials in the workspace
  int H;             // query heads
  int S;             // query rows
  int npairs;         // ceil(S / 128): Q-tile pairs per (batch, head)
  // Generalised problem (SURVEY.md 8f rows 2-3; reference: flash_attention_c/csrc/attn.cpp:121-124,182-183 for
  // Sq != Sk with a bottom-right aligned causal mask, csrc/archive_)/attn.cpp:61,375 for grouped K/V heads):
  int Sk;             // keys (== S for the reference's CuTe path; may be < S)
  int causal_off;     // Sk - S, negative when Sk < S: query row i sees keys j <= i + causal_off (rows i < -causal_off
                      // see none)
  int kv_group;       // query heads per K/V head (1 = MHA)
  // split-KV: the grid carries nsplit work items per Q-tile pair, each covering split_tiles KV tiles and writing a
  // normalised fp32 partial O plus its LSE; tfa_splitkv_combine merges them.  nsplit == 1: split_tiles = all.
  int nsplit;
  int split_tiles;
  long long part_stride;      // out_f32 elements between consecutive splits
  long long lse_part_stride;  // lse elements between consecutive splits
  // launch order (decode_work below): heads are taken in chunks of `head_chunk`; total (batch*head) count `BH`
  int head_chunk;
  int BH;
  int keyless_pairs;  // dense causal with Sq > Sk: the first Q-tile pairs of every (batch, head), which see no key
  int total_items;    // npairs * BH * nsplit
  float scale;        // softmax_scale
  float scale_log2;   // softmax_scale * log2(e)
  DebugRecord* dbg;
  // Variable length (VARLEN = true): batch entry b is the problem of rows [cu_q[b], cu_q[b+1]) of the packed q/out
  // and rows [cu_k[b], cu_k[b+1]) of the packed k/v; S is max_seqlen_q and Sk / causal_off are unused.  The arrays are
  // device memory, read by the kernel only; lse is (H, total_q).
  const int* cu_q;
  const int* cu_k;
  int total_q, total_k;
  // KV cache (MODE == kCache): q / out / lse are the dense (B, H, S) problem; sequence b attends to the first
  // cache_len(cache_seqlens[b]) + snew keys of its cache, whose key r lives at page_lookup(block_table, b, r).  The
  // K/V tensor maps are (D, page, Hkv, num_blocks).  Sk / causal_off are unused.
  // kVarlenCache: q / out / lse as varlen (cu_q, total_q; cu_k unused), K/V as kCache; sequence b attends to the
  // cache_lens() keys of its n_b = min(Sq_b, S) rows, with n_b appended keys when snew != 0 (a flag here).
  const int* cache_seqlens;
  const int* block_table;     // nullptr: contiguous cache, page = capacity
  long long bt_stride;
  int page, capacity, snew;
  // FP8 cache (kCacheFp8 / kVarlenCacheFp8): V element x8 stands for v_scale * x8; the epilogue folds it into 1/l.
  // (k_scale is folded into scale / scale_log2 by the host.)
  float v_scale;
};

template <int D>
struct FwdCfg {
  static_assert(D == 64 || D == 128, "head_dim must be 64 or 128");
  static constexpr int BM = 64;                     // rows per Q tile (one softmax warpgroup)
  static constexpr int BN = 128;                    // keys per KV tile
  static constexpr int SLABS = D / 64;              // 128-byte-wide swizzle slabs per tile row
  static constexpr int SLAB_BYTES = 128 * 128;      // 128 rows x 128 B
  static constexpr int TILE_BYTES = SLABS * SLAB_BYTES;   // 128 rows x D: the item's two Q tiles, or one K / V tile
  static constexpr int NSTAGE = (D == 128) ? 4 : 8; // K/V ring depth (tiles)
  static constexpr int NUM_BARS = 2 + 2 * NSTAGE;   // q_full, q_empty, kv_full[NSTAGE], kv_empty[NSTAGE]
  static constexpr int SMEM_BYTES = 1024 /*align slack*/ + TILE_BYTES /*Q*/ + TILE_BYTES /*O staging*/ +
                                    NSTAGE * TILE_BYTES + NUM_BARS * 8;
  static_assert(SMEM_BYTES <= 232448, "exceeds the 227 KB of shared memory a block may use");
  static constexpr int THREADS = 384;
};

// Shared-memory plan of the FP8-cache modes: the same Q and staging tiles, a 16-bit K/V ring of NSTAGE tiles, then a
// ring of NRAW raw e4m3 tiles (128 keys x D bytes, unswizzled, as TMA loads them), then the barriers: q_full, q_empty,
// kv_full / kv_empty[NSTAGE], raw_full / raw_empty[NRAW].  The D = 128 depths (4 + 2) come from an A/B of 4 + 2, 3 + 4
// and 2 + 6 on K1 / K3 of scripts/kvcache_fp8_bench.py (profiles/h100_kvcache_fp8.json; TFA_FP8_RING128 /
// TFA_FP8_RAW128 build the other pairs).  D = 64 keeps FwdCfg's 8-deep ring plus 4 raw tiles (197,840 B; 8 + 8 would
// fit too): no D = 64 workload was measured.
#ifndef TFA_FP8_RING128
#define TFA_FP8_RING128 4
#endif
#ifndef TFA_FP8_RAW128
#define TFA_FP8_RAW128 2
#endif
template <int D>
struct Fp8Cfg {
  using C = FwdCfg<D>;
  static constexpr int NSTAGE = (D == 128) ? TFA_FP8_RING128 : C::NSTAGE;
  static constexpr int RAW_BYTES = 128 * D;
  static constexpr int NRAW = (D == 128) ? TFA_FP8_RAW128 : 4;
  static constexpr int NUM_BARS = 2 + 2 * NSTAGE + 2 * NRAW;
  static constexpr int SMEM_BYTES =
      1024 + 2 * C::TILE_BYTES + NSTAGE * C::TILE_BYTES + NRAW * RAW_BYTES + NUM_BARS * 8;
  static_assert(SMEM_BYTES <= 232448, "exceeds the 227 KB of shared memory a block may use");
  static constexpr int CONVERTER_WARPS = 3;   // producer warps 1..3
};
// Shared-memory plan of kDenseFp8 and kVarlenFp8: Q (128 rows x D bytes), the 16-bit O staging of FwdCfg, then three rings of
// 128 x D-byte tiles -- K (filled by TMA, SWIZZLE_128B at D = 128, SWIZZLE_64B at D = 64), raw V (unswizzled, as TMA
// loads it) and V^T (D rows x 128 keys, SWIZZLE_128B, written by the converter) -- then the barriers: q_full, q_empty,
// k_full / k_empty[NK], raw_full / raw_empty[NRAW], vt_full / vt_empty[NVT].  Each ring has its own barriers, so each
// full barrier has one arrival count: 1 (TMA with its transaction bytes) for K and raw V, CONVERTER_WARPS for V^T.
// Tile j of the running tile count takes slot j % N of each ring.  The D = 128 depths (4 + 3 + 4) are the largest that
// fit with the K and V^T rings as deep as the 16-bit ring; they have not been A/B-measured against other splits, which
// TFA_FP8F_K128 / _RAW128 / _VT128 build.  D = 64 has room for 8 + 4 + 8.
#ifndef TFA_FP8F_K128
#define TFA_FP8F_K128 4
#endif
#ifndef TFA_FP8F_RAW128
#define TFA_FP8F_RAW128 3
#endif
#ifndef TFA_FP8F_VT128
#define TFA_FP8F_VT128 4
#endif
template <int D>
struct DenseFp8Cfg {
  using C = FwdCfg<D>;
  static constexpr int Q_BYTES = 128 * D;           // the item's two Q tiles
  static constexpr int TILE8 = 128 * D;             // one K, raw V or V^T tile
  static constexpr int NK = (D == 128) ? TFA_FP8F_K128 : 8;
  static constexpr int NRAW = (D == 128) ? TFA_FP8F_RAW128 : 4;
  static constexpr int NVT = (D == 128) ? TFA_FP8F_VT128 : 8;
  static constexpr int NUM_BARS = 2 + 2 * (NK + NRAW + NVT);
  static constexpr int SMEM_BYTES = 1024 + Q_BYTES + C::TILE_BYTES + (NK + NRAW + NVT) * TILE8 + NUM_BARS * 8;
  static_assert(SMEM_BYTES <= 232448, "exceeds the 227 KB of shared memory a block may use");
  static constexpr int CONVERTER_WARPS = 3;         // producer warps 1..3
};
template <int D, int MODE>
__host__ __device__ constexpr int fwd_smem_bytes() {
  return qkv8_mode(MODE) ? DenseFp8Cfg<D>::SMEM_BYTES : fp8_mode(MODE) ? Fp8Cfg<D>::SMEM_BYTES : FwdCfg<D>::SMEM_BYTES;
}

// 8 e4m3 codes (bytes of r, element 0 in the low byte of r.x) -> 8 16-bit values, exactly: the code's sign and its
// 7 exponent-mantissa bits placed at the top of the 16-bit type's exponent-mantissa field give x8 * 2^-(bias gap), and
// one exact multiply by 2^(bias gap) undoes it (subnormal codes included: they land on the 16-bit type's subnormals,
// which this multiply keeps).  The NaN codes 0x7f / 0xff give a NaN.
template <bool IS_BF16>
__device__ __forceinline__ uint4 widen_e4m3x8(uint2 r) {
  constexpr int SHIFT = IS_BF16 ? 4 : 7;                // 8 exponent bits (bf16) or 5 (fp16) above the mantissa
  constexpr uint32_t SCALE = IS_BF16 ? 0x7b807b80u : 0x5c005c00u;   // 2^120 (bf16), 2^8 (fp16), two lanes
  constexpr uint32_t NAN_MUL = IS_BF16 ? 0xffu : 0xf8u;              // 0x80 -> 0x7f80 / 0x7c00: exponent all ones
  uint32_t out[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const uint32_t w = i < 2 ? r.x : r.y;
    // bytes 2(i&1), 2(i&1)+1 of w -> the low bytes of the two 16-bit lanes
    const uint32_t y = __byte_perm(w, 0u, (i & 1) ? 0x4342u : 0x4140u);
    const uint32_t em = y & 0x007f007fu, sgn = y & 0x00800080u;
    uint32_t h = (sgn << 8) | (em << SHIFT), d;
    if constexpr (IS_BF16) asm("mul.rn.bf16x2 %0, %1, %2;" : "=r"(d) : "r"(h), "r"(SCALE));
    else asm("mul.rn.f16x2 %0, %1, %2;" : "=r"(d) : "r"(h), "r"(SCALE));
    const uint32_t nan = ((em + 0x00010001u) & 0x00800080u) * NAN_MUL;   // lanes whose code is 0x7f / 0xff
    out[i] = d | nan;
  }
  return make_uint4(out[0], out[1], out[2], out[3]);
}

// The converter of kDenseFp8 / kVarlenFp8, one unit u (0 <= u < 2 D) of a tile: keys [16 kc, 16 kc + 16) -- one 16-byte chunk of every
// V^T row -- x columns [4 dc, 4 dc + 4) of the raw tile at `raw` (128 keys x D bytes, row-major) into the V^T slot at
// `dst` (D rows x 128 keys, positions in fp8_vt_key order, SWIZZLE_128B).  Consecutive units take two chunks x 16
// columns per warp: its loads hit two rows per bank, its stores (8 lanes: four chunks x two rows) distinct bank groups.
// TAIL (kVarlenFp8): keys >= `valid` are written as zeros -- in a packed tile they are the next sequence's, any byte.
template <int D, bool TAIL = false>
__device__ __forceinline__ void vt_convert_unit(uint32_t raw, uint32_t dst, int u, int valid = 128) {
  constexpr int DC = D / 4;
  const int kc = 2 * (u / (2 * DC)) + (u & 1), dc = (u >> 1) % DC;
  uint32_t L[16];                                     // L[k] = columns 4 dc .. +3 of key 16 kc + k
#pragma unroll
  for (int k = 0; k < 16; ++k)
    asm volatile("ld.shared.u32 %0, [%1];" : "=r"(L[k]) : "r"(raw + (16 * kc + k) * D + 4 * dc));
  if constexpr (TAIL) {
    if (16 * kc + 16 > valid) {
#pragma unroll
      for (int k = 0; k < 16; ++k)
        if (16 * kc + k >= valid) L[k] = 0u;
    }
  }
  // row 4 dc + e, positions 16 kc + 4 x4 + x: key fp8_vt_key(16 kc + 4 x4 + x) = 16 kc + fp8_p_key(4 x4 + x), byte e
  // (one row at a time: the converter runs on kRegsProducerFp8 registers)
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    uint32_t W[4];
#pragma unroll
    for (int x4 = 0; x4 < 4; ++x4) {
      const uint32_t sel = e | ((e + 4) << 4);       // byte e of the first operand, then byte e of the second
      const uint32_t ab = __byte_perm(L[fp8_p_key(4 * x4 + 0)], L[fp8_p_key(4 * x4 + 1)], sel);
      const uint32_t cd = __byte_perm(L[fp8_p_key(4 * x4 + 2)], L[fp8_p_key(4 * x4 + 3)], sel);
      W[x4] = __byte_perm(ab, cd, 0x5410);
    }
    const int r = 4 * dc + e;                         // SWIZZLE_128B: chunk kc of row r at kc ^ (r & 7)
    asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};" ::"r"(dst + r * 128 + ((kc ^ (r & 7)) * 16)),
                 "r"(W[0]), "r"(W[1]), "r"(W[2]), "r"(W[3]) : "memory");
  }
}
// P (s[64], the fp32 accumulator layout of a 128-key tile) -> the A registers of its 4 k-steps of 32 keys, each
// thread's own values in fp8_p_key order.
__device__ __forceinline__ void pack_p_e4m3(const float* s, uint32_t* pf) {
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
    for (int r = 0; r < 4; ++r)
      pf[4 * kk + r] = pack_e4m3x4(s[16 * kk + fp8_pack_src(r, 0)], s[16 * kk + fp8_pack_src(r, 1)],
                                   s[16 * kk + fp8_pack_src(r, 2)], s[16 * kk + fp8_pack_src(r, 3)]);
  }
}

// watchdog call sites
enum : uint32_t { SITE_LOAD_EMPTY = 1, SITE_LOAD_Q = 2, SITE_MMA_Q = 3, SITE_MMA_K = 4, SITE_MMA_V = 5, SITE_CONV_RAW = 6 };

constexpr float kRescaleThresholdLog2 = 8.0f;  // lazy rescale: tolerate P up to 2^8
// Register re-allocation after the prologue.  setmaxnreg moves registers inside the CTA's OWN pool, which is
// what the launch allocated: 384 threads x 168 = 64512.  2 softmax warpgroups x 240 + 1 producer warpgroup x 24
// = 504 x 128 = 64512.
constexpr uint32_t kRegsSoftmax = 240;
constexpr uint32_t kRegsProducer = 24;
static_assert((2 * kRegsSoftmax + kRegsProducer) * 128 <= 384 * 168, "setmaxnreg budget exceeds the CTA register pool");
// The FP8-cache modes: the producer warpgroup widens every K/V tile, so it keeps more (2 x 232 + 40 = 504).
constexpr uint32_t kRegsSoftmaxFp8 = 232;
constexpr uint32_t kRegsProducerFp8 = 40;
static_assert((2 * kRegsSoftmaxFp8 + kRegsProducerFp8) * 128 <= 384 * 168,
              "setmaxnreg budget exceeds the CTA register pool");
// kDenseFp8: the converter transposes every V tile (sixteen 4-byte rows live per unit) and the softmax warpgroups hold
// P in 16 registers instead of 32 (2 x 224 + 56 = 504).
constexpr uint32_t kRegsSoftmaxDenseFp8 = 224;
constexpr uint32_t kRegsProducerDenseFp8 = 56;
static_assert((2 * kRegsSoftmaxDenseFp8 + kRegsProducerDenseFp8) * 128 <= 384 * 168,
              "setmaxnreg budget exceeds the CTA register pool");

// work item -> (batch*head, split, Q-tile pair).  CTAs are handed to SMs in blockIdx order (and the persistent kernel
// walks the same order), so this order IS the schedule.  Heads are taken in chunks of `head_chunk` (8) and INSIDE a
// chunk the order is (split, pair)-major, head-minor: all heads' heaviest item first, then their second heaviest, ...
// -- the tail is made of the lightest items of the last chunk, while the heads running concurrently (and with them the
// K/V working set in L2) stay what they were.  Host-callable so that a CPU test can check the mapping exhaustively
// (tests/test_abi.py).
__host__ __device__ __forceinline__ void decode_work(int block, int npairs, int nsplit, int head_chunk, int BH,
                                                     int& bh, int& split, int& pr) {
  const int per_bh = npairs * nsplit;                 // items per (batch, head)
  const int per_chunk = head_chunk * per_bh;
  const int chunk = block / per_chunk;
  const int r = block - chunk * per_chunk;
  const int g = min(head_chunk, BH - chunk * head_chunk);   // heads in this chunk (the last one may be short)
  const int sp = r / g;                               // (split, pair) index, heaviest pair first
  bh = chunk * head_chunk + (r - sp * g);
  split = sp / npairs;
  pr = npairs - 1 - (sp - split * npairs);
}

// One work item: both Q tiles walk the same KV tiles [jb, jb + n); rows a tile does not see are masked.
// q0 / k0 are the sequence's first row in the (packed) q and k/v tensors, Sq / Sk / coff its own lengths and causal
// offset: the whole tensor's (q0 = k0 = 0) for kDense, the cached length for kCache.  `live`: the item has rows to
// write -- every dense and cache item, and a packed item inside its sequence.  The producer loads an item iff n > 0,
// the softmax warpgroups wait on its barriers iff n > 0: n > 0 implies live.  A live item with n == 0 writes O = 0 and
// LSE = +inf (its rows see no key), or in a split-KV partial only LSE = -inf (its split holds none of their keys).
struct Item {
  int bh, bidx, hidx, hkv, split, jb, row0, n;
  int q0, k0, Sq, Sk, coff;
  bool live;
};
template <bool CAUSAL, int MODE>
__device__ __forceinline__ Item decode_item(int item, const FwdParams& p) {
  constexpr int M = base_mode(MODE);
  constexpr bool VARLEN = M == kVarlen;
  constexpr bool QPACK = M == kVarlen || M == kVarlenCache;          // packed queries: items past a sequence skipped
  Item w;
  int pr;
  // dense: the items of the Q-tile pairs whose rows see no key follow all others, in decode_work order of their own.
  // Interleaved with the rest, they would give some persistent CTAs up to twice the average share of keyed items.
  const int keyless = M == kDense ? p.keyless_pairs : 0;
  const int keyed_items = (p.npairs - keyless) * p.nsplit * p.BH;
  if (keyless == 0 || item < keyed_items) {
    decode_work(item, p.npairs - keyless, p.nsplit, p.head_chunk, p.BH, w.bh, w.split, pr);
    pr += keyless;
  } else {
    decode_work(item - keyed_items, keyless, p.nsplit, p.head_chunk, p.BH, w.bh, w.split, pr);
  }
  w.bidx = w.bh / p.H;
  w.hidx = w.bh - w.bidx * p.H;
  w.hkv = w.hidx / p.kv_group;
  w.row0 = pr * 128;
  w.jb = w.split * p.split_tiles;
  if constexpr (VARLEN) {
    // clamped to the packed tensors: whatever cu_seqlens holds, no row outside [0, total) is read or written
    const int q0 = min(max(__ldg(p.cu_q + w.bidx), 0), p.total_q);
    const int q1 = min(max(__ldg(p.cu_q + w.bidx + 1), 0), p.total_q);
    const int k0 = min(max(__ldg(p.cu_k + w.bidx), 0), p.total_k);
    const int k1 = min(max(__ldg(p.cu_k + w.bidx + 1), 0), p.total_k);
    w.q0 = q0;
    w.k0 = k0;
    w.Sq = max(q1 - q0, 0);
    w.Sk = max(k1 - k0, 0);
    w.coff = w.Sk - w.Sq;           // may be negative: the sequence's first rows see no key
    // kVarlenFp8 stores only the rows the header promises, the first max_seqlen_q = S (the grid covers up to the next
    // multiple of 128); the causal offset stays that of all Sq_b rows, as for kVarlen
    if constexpr (MODE == kVarlenFp8) w.Sq = min(w.Sq, p.S);
  } else if constexpr (M == kCache) {
    w.q0 = 0;
    w.k0 = 0;
    w.Sq = p.S;
    w.Sk = cache_len(__ldg(p.cache_seqlens + w.bidx), p.capacity, p.snew) + p.snew;
    w.coff = w.Sk - w.Sq;           // may be negative, as for varlen
  } else if constexpr (M == kVarlenCache) {
    // queries as varlen, but only the first S = max_seqlen_q rows: the grid covers no more, and the keys appended
    // for the sequence are those rows' own
    const int q0 = min(max(__ldg(p.cu_q + w.bidx), 0), p.total_q);
    const int q1 = min(max(__ldg(p.cu_q + w.bidx + 1), 0), p.total_q);
    w.q0 = q0;
    w.k0 = 0;
    w.Sq = min(max(q1 - q0, 0), p.S);
    int L;
    cache_lens(__ldg(p.cache_seqlens + w.bidx), p.capacity, p.snew ? w.Sq : 0, L, w.Sk);
    w.coff = w.Sk - w.Sq;
  } else {
    w.q0 = 0;
    w.k0 = 0;
    w.Sq = p.S;
    w.Sk = p.Sk;
    w.coff = p.causal_off;
  }
  const int nkv_total = (w.Sk + 127) >> 7;
  // causal: the item's last row sees keys <= last (none when last < 0)
  const int last = w.row0 + 127 + w.coff;
  const int nfull = CAUSAL ? (last < 0 ? 0 : min(nkv_total, last / 128 + 1)) : nkv_total;
  w.n = max(0, min(nfull - w.jb, p.split_tiles));   // 0: rows that see no key, or a split past the causal diagonal
  // every item writes its rows (a split without tiles their LSE), so the combine can read every split; only a packed
  // item past its sequence's end has none
  w.live = !QPACK || w.row0 < w.Sq;
  if (!w.live) w.n = 0;              // past the sequence's end: the producer must skip it as the consumers do
  return w;
}

template <int D, bool CAUSAL, bool IS_BF16, bool OUT_F32, bool PERSIST, int MODE>
__global__ void __launch_bounds__(384, 1)
fa_fwd_sm90_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                   const __grid_constant__ CUtensorMap tmV, const FwdParams p) {
  constexpr int M = base_mode(MODE);
  constexpr bool FP8 = fp8_mode(MODE);                          // K/V from an e4m3 cache, widened by the converter
  constexpr bool QPACK = M == kVarlen || M == kVarlenCache;     // q / out / lse packed as varlen
  constexpr bool PAGED = M == kCache || M == kVarlenCache;      // K/V from a (paged) cache
  using C = FwdCfg<D>;
  using F = Fp8Cfg<D>;
  constexpr int TILE = C::TILE_BYTES;
  constexpr int NSTAGE = FP8 ? F::NSTAGE : C::NSTAGE;          // 16-bit K/V ring depth
  constexpr bool DF8 = qkv8_mode(MODE);                         // Q, K, V in e4m3 and 8-bit wgmma
  using F8 = DenseFp8Cfg<D>;

  extern __shared__ uint8_t smem_raw[];
  // SWIZZLE_128B operands need 1024-byte alignment (the swizzle is a function of address bits 7..9)
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;                       // the item's two Q tiles: rows [0,64) tile 0, [64,128) tile 1
  uint8_t* sStg = smem + (DF8 ? F8::Q_BYTES : TILE);   // epilogue staging, 128 rows x D 16-bit
  uint8_t* sKV = smem + 2 * TILE;           // NSTAGE tiles
  // FP8: the raw e4m3 ring sits between the K/V ring and the barriers, its barriers after the others
  uint8_t* sRaw = sKV + NSTAGE * TILE;      // [NRAW] tiles of 128 keys x D bytes
  // kDenseFp8: the K, raw V and V^T rings after Q and the staging, their barriers after those
  uint8_t* sK8 = smem + F8::Q_BYTES + TILE;
  uint8_t* sRaw8 = sK8 + F8::NK * F8::TILE8;
  uint8_t* sVt = sRaw8 + F8::NRAW * F8::TILE8;
  uint64_t* bars = reinterpret_cast<uint64_t*>(DF8 ? sVt + F8::NVT * F8::TILE8
                                                   : sKV + NSTAGE * TILE + (FP8 ? F::NRAW * F::RAW_BYTES : 0));
  uint64_t* q_full = bars;
  uint64_t* q_empty = bars + 1;
  uint64_t* kv_full = bars + 2;             // [NSTAGE]
  uint64_t* kv_empty = kv_full + NSTAGE;    // [NSTAGE]
  uint64_t* raw_full = kv_empty + NSTAGE;   // [NRAW] (FP8 only)
  uint64_t* raw_empty = raw_full + F::NRAW; // [NRAW]
  uint64_t* k_full = bars + 2;              // kDenseFp8: [NK]
  uint64_t* k_empty = k_full + F8::NK;      // [NK]
  uint64_t* raw8_full = k_empty + F8::NK;   // [NRAW]
  uint64_t* raw8_empty = raw8_full + F8::NRAW;
  uint64_t* vt_full = raw8_empty + F8::NRAW;   // [NVT]
  uint64_t* vt_empty = vt_full + F8::NVT;      // [NVT]

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int first = static_cast<int>(blockIdx.x);
  const int stride = PERSIST ? static_cast<int>(gridDim.x) : p.total_items;
  if (!PERSIST && !decode_item<CAUSAL, MODE>(first, p).live) return;   // CTA-uniform

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmK);
    tma_prefetch_desc(&tmV);
    mbar_init(q_full, 1);
    mbar_init(q_empty, 8);             // one arrival per softmax warp
    if constexpr (DF8) {
      for (int i = 0; i < F8::NK; ++i) {
        mbar_init(&k_full[i], 1);
        mbar_init(&k_empty[i], 8);
      }
      for (int i = 0; i < F8::NRAW; ++i) {
        mbar_init(&raw8_full[i], 1);
        mbar_init(&raw8_empty[i], F8::CONVERTER_WARPS);
      }
      for (int i = 0; i < F8::NVT; ++i) {
        mbar_init(&vt_full[i], F8::CONVERTER_WARPS);       // one arrival per converter warp
        mbar_init(&vt_empty[i], 8);
      }
    } else {
      for (int i = 0; i < NSTAGE; ++i) {
        mbar_init(&kv_full[i], FP8 ? F::CONVERTER_WARPS : 1);   // FP8: one arrival per converter warp
        mbar_init(&kv_empty[i], 8);
      }
      if constexpr (FP8) {
        for (int i = 0; i < F::NRAW; ++i) {
          mbar_init(&raw_full[i], 1);
          mbar_init(&raw_empty[i], F::CONVERTER_WARPS);
        }
      }
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp < 4) {
    // =========================== TMA producer ===========================
    setmaxnreg_dec<DF8 ? kRegsProducerDenseFp8 : FP8 ? kRegsProducerFp8 : kRegsProducer>();
    if constexpr (DF8) {
      if (warp > 0) {
        // ---- the converter (warps 1..3): raw V tile (128 keys x D bytes) -> V^T slot (D rows x 128 keys, keys in
        // fp8_vt_key order, SWIZZLE_128B), walking the TMA lane's tiles.  Dense: keys past Sk arrive as TMA's zero fill.
        // Packed: they are the next sequence's keys, any byte, NaN codes included (P = 0 does not cancel 0 * NaN), so
        // they are written as zeros, which also makes a sequence's result that of the dense call on it alone. ----
        const int ct = threadIdx.x - 32;                          // 0 .. 95
        uint32_t tile = 0;
        for (int item = first; item < p.total_items; item += stride) {
          const Item w = decode_item<CAUSAL, MODE>(item, p);
#pragma unroll 1
          for (int j = 0; j < w.n; ++j, ++tile) {
            const uint32_t rslot = tile % F8::NRAW, vslot = tile % F8::NVT;
            mbar_wait(&raw8_full[rslot], (tile / F8::NRAW) & 1, p.dbg, SITE_CONV_RAW, tile);
            mbar_wait(&vt_empty[vslot], ((tile / F8::NVT) & 1) ^ 1, p.dbg, SITE_LOAD_EMPTY, tile);
            const uint32_t raw = smem_u32(sRaw8) + rslot * F8::TILE8;
            const uint32_t dst = smem_u32(sVt) + vslot * F8::TILE8;
            if constexpr (QPACK) {
              const int valid = w.Sk - (w.jb + j) * C::BN;
#pragma unroll 1
              for (int u = ct; u < 2 * D; u += 32 * F8::CONVERTER_WARPS) vt_convert_unit<D, true>(raw, dst, u, valid);
            } else {
#pragma unroll 1
              for (int u = ct; u < 2 * D; u += 32 * F8::CONVERTER_WARPS) vt_convert_unit<D>(raw, dst, u);
            }
            fence_proxy_async_smem();                             // generic-proxy stores -> the wgmma's operand reads
            __syncwarp();
            if (lane == 0) {
              mbar_arrive(&vt_full[vslot]);
              mbar_arrive(&raw8_empty[rslot]);
            }
          }
        }
      } else if (lane == 0) {
        // ---- the TMA lane: the item's Q (one 128-row box), then per KV tile K into the K ring and V raw ----
        uint32_t tile = 0;     // running KV tile (never reset between items)
        uint32_t qcnt = 0;
        for (int item = first; item < p.total_items; item += stride) {
          const Item w = decode_item<CAUSAL, MODE>(item, p);
          if (w.n == 0) continue;
          if (qcnt > 0) mbar_wait(q_empty, (qcnt - 1) & 1, p.dbg, SITE_LOAD_Q, qcnt);
          ++qcnt;
          mbar_arrive_expect_tx(q_full, F8::Q_BYTES);
          // packed (kVarlenFp8): the tensors are one batch entry, the sequence starts at row q0 / k0.  Rows a box takes
          // in past the sequence's end are never stored (queries) or get -inf from the edge mask (keys; their V^T
          // entries the converter writes as zeros)
          int qy = w.row0, k0 = 0, wz = w.bidx;
          if constexpr (QPACK) {
            qy += w.q0;
            k0 = w.k0;
            wz = 0;
          }
          tma_load_4d(sQ, &tmQ, q_full, 0, qy, w.hidx, wz);
          for (int j = 0; j < w.n; ++j, ++tile) {
            const int ky = k0 + (w.jb + j) * C::BN;
            const uint32_t kslot = tile % F8::NK, rslot = tile % F8::NRAW;
            mbar_wait(&k_empty[kslot], ((tile / F8::NK) & 1) ^ 1, p.dbg, SITE_LOAD_EMPTY, tile);
            mbar_arrive_expect_tx(&k_full[kslot], F8::TILE8);
            tma_load_4d(sK8 + kslot * F8::TILE8, &tmK, &k_full[kslot], 0, ky, w.hkv, wz);
            mbar_wait(&raw8_empty[rslot], ((tile / F8::NRAW) & 1) ^ 1, p.dbg, SITE_LOAD_EMPTY, tile);
            mbar_arrive_expect_tx(&raw8_full[rslot], F8::TILE8);
            tma_load_4d(sRaw8 + rslot * F8::TILE8, &tmV, &raw8_full[rslot], 0, ky, w.hkv, wz);
          }
        }
      }
      return;
    }
    if constexpr (FP8) {
      if (warp > 0) {
        // ---- the converter (warps 1..3): raw ring entry -> 16-bit K/V ring slot, walking the TMA lane's entries ----
        uint32_t ent = 0;
        const int ct = threadIdx.x - 32;                          // 0 .. 95
        for (int item = first; item < p.total_items; item += stride) {
          const Item w = decode_item<CAUSAL, MODE>(item, p);
          if (w.n == 0) continue;
          for (int j = 0; j < w.n; ++j) {
            // rows at or past the sequence's keys become zeros: a slot past K_b may hold any byte, NaN codes included,
            // and P = 0 does not cancel 0 * NaN in the PV product (the 16-bit modes' zero_v_tail)
            const int valid = w.Sk - (w.jb + j) * C::BN;
#pragma unroll 1
            for (int kv = 0; kv < 2; ++kv, ++ent) {
              const uint32_t slot = ent % NSTAGE, rslot = ent % F::NRAW;
              mbar_wait(&raw_full[rslot], (ent / F::NRAW) & 1, p.dbg, SITE_CONV_RAW, ent);
              mbar_wait(&kv_empty[slot], ((ent / NSTAGE) & 1) ^ 1, p.dbg, SITE_LOAD_EMPTY, ent);
              // 32-bit shared-memory addresses: this warpgroup runs on kRegsProducerFp8 registers
              const uint32_t raw = smem_u32(sRaw) + rslot * F::RAW_BYTES;
              const uint32_t dst = smem_u32(sKV) + slot * TILE;
              constexpr int CPR = D / 8;                          // 16-byte output chunks per key row
#pragma unroll 2
              for (int idx = ct; idx < C::BN * CPR; idx += 32 * F::CONVERTER_WARPS) {
                const int r = idx / CPR, c = idx % CPR;           // key row, chunk of 8 elements
                uint4 v = make_uint4(0u, 0u, 0u, 0u);
                if (r < valid) {
                  uint2 x;
                  asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(x.x), "=r"(x.y) : "r"(raw + idx * 8));
                  v = widen_e4m3x8<IS_BF16>(x);
                }
                // SWIZZLE_128B, as TMA lays out a 16-bit tile: 64-column slabs, chunk c of row r at (c ^ r) & 7
                asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};"
                             ::"r"(dst + (c / 8) * C::SLAB_BYTES + r * 128 + (((c & 7) ^ (r & 7)) * 16)),
                               "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
              }
              fence_proxy_async_smem();                           // generic-proxy stores -> the wgmma's operand reads
              __syncwarp();
              if (lane == 0) {
                mbar_arrive(&kv_full[slot]);
                mbar_arrive(&raw_empty[rslot]);
              }
            }
          }
        }
        return;
      }
    }
    if (warp == 0 && lane == 0) {
      uint32_t ent = 0;      // running K/V ring entry (K_j and V_j of every item in turn; never reset between items)
      uint32_t qcnt = 0;     // items loaded
      for (int item = first; item < p.total_items; item += stride) {
        const Item w = decode_item<CAUSAL, MODE>(item, p);
        if (w.n == 0) continue;
        if (qcnt > 0) mbar_wait(q_empty, (qcnt - 1) & 1, p.dbg, SITE_LOAD_Q, qcnt);
        ++qcnt;
        mbar_arrive_expect_tx(q_full, TILE);
        // varlen: the packed tensors are one batch entry; rows of the next sequence a box takes in are never stored
        // (queries) or masked (keys)
        const int wz = QPACK ? 0 : w.bidx;
#pragma unroll
        for (int sl = 0; sl < C::SLABS; ++sl)
          tma_load_4d(sQ + sl * C::SLAB_BYTES, &tmQ, q_full, sl * 64, w.q0 + w.row0, w.hidx, wz);
        for (int j = 0; j < w.n; ++j) {
          // cache: the tile's 128 keys lie in one page (page % 128 == 0, or one page per sequence)
          int ky = w.k0 + (w.jb + j) * C::BN, kw = wz;
          if constexpr (PAGED) page_lookup(p.block_table, p.bt_stride, w.bidx, ky, p.page, kw, ky);
#pragma unroll
          for (int kv = 0; kv < 2; ++kv, ++ent) {
            const CUtensorMap* tm = kv ? &tmV : &tmK;
            if constexpr (FP8) {
              // one unswizzled box of 128 keys x D bytes into the raw ring; the converter fills the K/V slot
              const uint32_t rslot = ent % F::NRAW;
              mbar_wait(&raw_empty[rslot], ((ent / F::NRAW) & 1) ^ 1, p.dbg, SITE_LOAD_EMPTY, ent);
              mbar_arrive_expect_tx(&raw_full[rslot], F::RAW_BYTES);
              tma_load_4d(sRaw + rslot * F::RAW_BYTES, tm, &raw_full[rslot], 0, ky, w.hkv, kw);
            } else {
              const uint32_t slot = ent % NSTAGE;
              mbar_wait(&kv_empty[slot], ((ent / NSTAGE) & 1) ^ 1, p.dbg, SITE_LOAD_EMPTY, ent);
              mbar_arrive_expect_tx(&kv_full[slot], TILE);
#pragma unroll
              for (int sl = 0; sl < C::SLABS; ++sl)
                tma_load_4d(sKV + slot * TILE + sl * C::SLAB_BYTES, tm, &kv_full[slot], sl * 64, ky, w.hkv, kw);
            }
          }
        }
      }
    }
    return;
  }

  // ================= softmax / wgmma / epilogue warpgroup t =================
  setmaxnreg_inc<DF8 ? kRegsSoftmaxDenseFp8 : FP8 ? kRegsSoftmaxFp8 : kRegsSoftmax>();
  using MmaS = Wgmma<128, IS_BF16>;
  using MmaO = Wgmma<D, IS_BF16>;
  const int t = (warp >> 2) - 1;                 // Q tile
  const int wq = warp & 3;                       // warp inside the warpgroup: rows [16 wq, 16 wq + 16) of the tile
  const int g = lane >> 2, tq = lane & 3;        // this thread: rows 16 wq + g and + 8, columns 8 i + 2 tq (+1)
  const int r_lo = t * 64 + wq * 16 + g;         // row inside the item (0..127); r_hi = r_lo + 8
  const float c = p.scale_log2;
  const uint32_t sQ_addr = smem_u32(sQ) + t * 64 * 128;   // this tile's rows inside each slab
  const uint32_t sKV_addr = smem_u32(sKV);

  uint32_t ent = 0;        // K/V ring entry of K_0 of the current item (same sequence as the producer's)
  uint32_t qcnt = 0;
  for (int item = first; item < p.total_items; item += stride) {
    const Item w = decode_item<CAUSAL, MODE>(item, p);
    const int n = w.n;
    if (!w.live) continue;
    const int S = w.Sq, Sk = w.Sk, coff = w.coff;
    const int row_lo = w.row0 + r_lo, row_hi = row_lo + 8;    // query rows of the sequence

    // S = Q K^T over D/16 k-steps; K-major operands advance 32 B per k-step inside a slab, one slab per 4 k-steps
    // kDenseFp8: D/32 k-steps of 32 bytes inside the tile's D-byte rows (128-byte swizzle at D = 128, 64-byte at 64)
    auto issue_S = [&](float* s, uint32_t kslot) {
      if constexpr (DF8) {
        const uint32_t q_addr = smem_u32(sQ) + t * 64 * D, k_addr = smem_u32(sK8) + kslot * F8::TILE8;
#pragma unroll
        for (int kk = 0; kk < D / 32; ++kk) {
          const uint64_t dq = D == 128 ? gmma_desc(q_addr + kk * 32, 16, 1024) : gmma_desc_sw64(q_addr + kk * 32, 512);
          const uint64_t dk = D == 128 ? gmma_desc(k_addr + kk * 32, 16, 1024) : gmma_desc_sw64(k_addr + kk * 32, 512);
          WgmmaE4m3<128>::ss(s, dq, dk, kk > 0 ? 1u : 0u);
        }
      } else {
        const uint32_t k_addr = sKV_addr + kslot * TILE;
#pragma unroll
        for (int kk = 0; kk < D / 16; ++kk) {
          const uint32_t off = (kk / 4) * C::SLAB_BYTES + (kk % 4) * 32;
          MmaS::template ss<0>(s, gmma_desc(sQ_addr + off, 16, 1024), gmma_desc(k_addr + off, 16, 1024), kk > 0 ? 1u : 0u);
        }
      }
      wgmma_commit();
    };
    // O += P V over 8 k-steps of 16 keys; V is MN-major: 16 key rows = 2048 B per k-step, LBO = next 64-column slab
    // kDenseFp8: 4 k-steps of 32 keys; V^T is K-major, 32 B per k-step inside its 128-byte rows
    auto issue_PV = [&](float* o, const uint32_t* pf, uint32_t vslot, bool acc) {
      if constexpr (DF8) {
        const uint32_t vt_addr = smem_u32(sVt) + vslot * F8::TILE8;
#pragma unroll
        for (int kk = 0; kk < C::BN / 32; ++kk)
          WgmmaE4m3<D>::rs(o, pf + 4 * kk, gmma_desc(vt_addr + kk * 32, 16, 1024), (acc || kk > 0) ? 1u : 0u);
      } else {
        const uint32_t v_addr = sKV_addr + vslot * TILE;
#pragma unroll
        for (int kk = 0; kk < C::BN / 16; ++kk)
          MmaO::rs(o, pf + 4 * kk, gmma_desc(v_addr + kk * 2048, C::SLAB_BYTES, 1024), (acc || kk > 0) ? 1u : 0u);
      }
      wgmma_commit();
    };
    auto release = [&](uint64_t* bar) {
      __syncwarp();
      if (lane == 0) mbar_arrive(bar);
    };
    // cache: the slots of a page past the sequence's keys may hold anything, NaN included, and P = 0 does not cancel
    // 0 * NaN in the PV product.  So before PV reads the tile holding key Sk - 1, this warpgroup zeroes the V rows
    // [Sk, tile end) in shared memory (whole 128-byte swizzle rows of each slab, so the swizzle does not matter).  Both
    // warpgroups write the same zeros; the slot is released only after both have read it.  Between the kv_full wait
    // and the release, so the producer cannot refill the slot under the stores (scripts/protocol_model.py).
    // FP8: the converter wrote those rows as zeros already.
    auto zero_v_tail = [&](uint32_t vslot, int jt) {
      if constexpr (PAGED && !FP8) {
        const int valid = Sk - (w.jb + jt) * C::BN;          // warpgroup-uniform
        if (valid < C::BN) {
          uint8_t* vt = sKV + vslot * TILE;
          const uint4 z = make_uint4(0u, 0u, 0u, 0u);
          for (int idx = valid * 8 + (threadIdx.x & 127); idx < C::BN * 8; idx += 128) {
#pragma unroll
            for (int sl = 0; sl < C::SLABS; ++sl) *reinterpret_cast<uint4*>(vt + sl * C::SLAB_BYTES + idx * 16) = z;
          }
          fence_proxy_async_smem();                          // generic-proxy stores -> the wgmma's operand reads
          named_bar_sync(1 + t, 128);
        }
      }
    };

    float s[64];             // S tile: 16 column groups of 8 keys x {row_lo: [0],[1], row_hi: [2],[3]}
    float o[D / 2];          // O tile, same layout over D columns
    uint32_t pf[DF8 ? 16 : 32];   // P as the A operand: 8 k-steps x 4 registers of 16-bit pairs (e4m3: 4 x 4 of e4m3x4)
    float m_lo = 0.f, m_hi = 0.f;     // reference max the exponentials are taken against (raw score units)
    float l_lo = 0.f, l_hi = 0.f;     // this thread's part of the running sum of exp2((s - m) * c)
#pragma unroll
    for (int i = 0; i < D / 2; ++i) o[i] = 0.f;

    // mask + row max + lazy rescale decision + P = exp2(s*c - m*c) (fp32, in s) + row sums
    // returns alpha for (lo, hi) when O must be rescaled (rare), else {1, 1}
    auto softmax = [&](int j, bool& rescale, float& a_lo, float& a_hi) {
      const int col0 = (w.jb + j) * C::BN;
      const bool edge = (col0 + C::BN > Sk) || (CAUSAL && col0 + C::BN - 1 > w.row0 + t * 64 + coff);
      if (edge) {     // tiles crossing the causal diagonal or the end of the keys (warpgroup-uniform)
        const int lim_lo = (CAUSAL ? min(Sk, row_lo + coff + 1) : Sk) - col0;
        const int lim_hi = (CAUSAL ? min(Sk, row_hi + coff + 1) : Sk) - col0;
#pragma unroll
        for (int i = 0; i < 16; ++i) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int col = 8 * i + 2 * tq + e;
            if (col >= lim_lo) s[4 * i + e] = -INFINITY;
            if (col >= lim_hi) s[4 * i + 2 + e] = -INFINITY;
          }
        }
      }
      float mx_lo = -INFINITY, mx_hi = -INFINITY;
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        mx_lo = fmaxf(mx_lo, fmaxf(s[4 * i], s[4 * i + 1]));
        mx_hi = fmaxf(mx_hi, fmaxf(s[4 * i + 2], s[4 * i + 3]));
      }
#pragma unroll
      for (int d = 1; d <= 2; d <<= 1) {
        mx_lo = fmaxf(mx_lo, __shfl_xor_sync(0xffffffffu, mx_lo, d));
        mx_hi = fmaxf(mx_hi, __shfl_xor_sync(0xffffffffu, mx_hi, d));
      }
      a_lo = a_hi = 1.f;
      rescale = false;
      if (j == 0) {
        m_lo = fmaxf(mx_lo, -1.0e30f);             // a fully masked row (split-KV) must not give -inf
        m_hi = fmaxf(mx_hi, -1.0e30f);
      } else {
        // lazy rescale of l and O: only when the row max moved by more than 2^8 (warp-uniform branch, rare)
        const bool n_lo = (mx_lo - m_lo) * c > kRescaleThresholdLog2;
        const bool n_hi = (mx_hi - m_hi) * c > kRescaleThresholdLog2;
        if (__any_sync(0xffffffffu, n_lo || n_hi)) {
          rescale = true;
          if (n_lo) { a_lo = ex2_approx((m_lo - mx_lo) * c); m_lo = mx_lo; }
          if (n_hi) { a_hi = ex2_approx((m_hi - mx_hi) * c); m_hi = mx_hi; }
          l_lo *= a_lo;
          l_hi *= a_hi;
        }
      }
      const float nm_lo = -m_lo * c, nm_hi = -m_hi * c;
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        s[4 * i + 0] = ex2_approx(fmaf(s[4 * i + 0], c, nm_lo));
        s[4 * i + 1] = ex2_approx(fmaf(s[4 * i + 1], c, nm_lo));
        s[4 * i + 2] = ex2_approx(fmaf(s[4 * i + 2], c, nm_hi));
        s[4 * i + 3] = ex2_approx(fmaf(s[4 * i + 3], c, nm_hi));
        l_lo += s[4 * i + 0] + s[4 * i + 1];      // l sums fp32 P, before the 16-bit rounding
        l_hi += s[4 * i + 2] + s[4 * i + 3];
      }
    };
    // P (fp32 accumulator layout) -> A-operand registers: k-step kk = column groups 2kk, 2kk+1
    // kDenseFp8: P <= 2^8 < 448 (the lazy rescale's bound) is in e4m3 range
    auto pack_P = [&]() {
      if constexpr (DF8) {
        pack_p_e4m3(s, pf);
      } else {
#pragma unroll
        for (int kk = 0; kk < 8; ++kk) {
          pf[4 * kk + 0] = pack_16x2<IS_BF16>(s[8 * kk + 0], s[8 * kk + 1]);
          pf[4 * kk + 1] = pack_16x2<IS_BF16>(s[8 * kk + 2], s[8 * kk + 3]);
          pf[4 * kk + 2] = pack_16x2<IS_BF16>(s[8 * kk + 4], s[8 * kk + 5]);
          pf[4 * kk + 3] = pack_16x2<IS_BF16>(s[8 * kk + 6], s[8 * kk + 7]);
        }
      }
    };

    // An item without tiles waits on no barrier: its rows get O = 0 and LSE = +inf (a split-KV partial: LSE = -inf).
    if (DF8 && n > 0) {
      // kDenseFp8: K_j on k_full[(ent + j) % NK], V^T_j on vt_full[(ent + j) % NVT]; ent counts earlier items' tiles
      mbar_wait(q_full, qcnt & 1, p.dbg, SITE_MMA_Q, qcnt);
      ++qcnt;
      {
        const uint32_t kslot = ent % F8::NK;
        mbar_wait(&k_full[kslot], (ent / F8::NK) & 1, p.dbg, SITE_MMA_K, ent);
        wgmma_fence();
        issue_S(s, kslot);
        wgmma_wait<0>();
        reg_fence(s);
        release(&k_empty[kslot]);
        if (n == 1) release(q_empty);
        bool rs;
        float a0, a1;
        softmax(0, rs, a0, a1);
        pack_P();
      }
      for (int j = 1; j < n; ++j) {
        const uint32_t ek = ent + j, ev = ent + j - 1;
        const uint32_t kslot = ek % F8::NK, vslot = ev % F8::NVT;
        mbar_wait(&k_full[kslot], (ek / F8::NK) & 1, p.dbg, SITE_MMA_K, ek);
        wgmma_fence();
        issue_S(s, kslot);
        mbar_wait(&vt_full[vslot], (ev / F8::NVT) & 1, p.dbg, SITE_MMA_V, ev);
        issue_PV(o, pf, vslot, j > 1);
        wgmma_wait<1>();                               // S_j done
        reg_fence(s);
        release(&k_empty[kslot]);
        if (j == n - 1) release(q_empty);
        bool rs;
        float a_lo, a_hi;
        softmax(j, rs, a_lo, a_hi);
        wgmma_wait<0>();                               // PV_{j-1} done: O and P registers are ours again
        reg_fence(o);
        release(&vt_empty[vslot]);
        if (rs) {
#pragma unroll
          for (int i = 0; i < D / 8; ++i) {
            o[4 * i + 0] *= a_lo; o[4 * i + 1] *= a_lo;
            o[4 * i + 2] *= a_hi; o[4 * i + 3] *= a_hi;
          }
        }
        pack_P();
      }
      {
        const uint32_t ev = ent + n - 1, vslot = ev % F8::NVT;
        mbar_wait(&vt_full[vslot], (ev / F8::NVT) & 1, p.dbg, SITE_MMA_V, ev);
        wgmma_fence();
        issue_PV(o, pf, vslot, n > 1);
        wgmma_wait<0>();
        reg_fence(o);
        release(&vt_empty[vslot]);
      }
      ent += n;
    } else if (n > 0) {
      mbar_wait(q_full, qcnt & 1, p.dbg, SITE_MMA_Q, qcnt);
      ++qcnt;
      // ---- KV tile 0 ----
      {
        const uint32_t kslot = ent % NSTAGE;
        mbar_wait(&kv_full[kslot], (ent / NSTAGE) & 1, p.dbg, SITE_MMA_K, ent);
        wgmma_fence();
        issue_S(s, kslot);
        wgmma_wait<0>();
        reg_fence(s);
        release(&kv_empty[kslot]);
        if (n == 1) release(q_empty);
        bool rs;
        float a0, a1;
        softmax(0, rs, a0, a1);
        pack_P();
      }
      // ---- KV tiles 1 .. n-1: S_j and PV_{j-1} in flight together ----
      for (int j = 1; j < n; ++j) {
        const uint32_t ek = ent + 2 * j, ev = ent + 2 * j - 1;
        const uint32_t kslot = ek % NSTAGE, vslot = ev % NSTAGE;
        mbar_wait(&kv_full[kslot], (ek / NSTAGE) & 1, p.dbg, SITE_MMA_K, ek);
        wgmma_fence();
        issue_S(s, kslot);
        mbar_wait(&kv_full[vslot], (ev / NSTAGE) & 1, p.dbg, SITE_MMA_V, ev);
        zero_v_tail(vslot, j - 1);
        issue_PV(o, pf, vslot, j > 1);
        wgmma_wait<1>();                               // S_j done
        reg_fence(s);
        release(&kv_empty[kslot]);
        if (j == n - 1) release(q_empty);
        bool rs;
        float a_lo, a_hi;
        softmax(j, rs, a_lo, a_hi);
        wgmma_wait<0>();                               // PV_{j-1} done: O and P registers are ours again
        reg_fence(o);
        release(&kv_empty[vslot]);
        if (rs) {
#pragma unroll
          for (int i = 0; i < D / 8; ++i) {
            o[4 * i + 0] *= a_lo; o[4 * i + 1] *= a_lo;
            o[4 * i + 2] *= a_hi; o[4 * i + 3] *= a_hi;
          }
        }
        pack_P();
      }
      {
        const uint32_t ev = ent + 2 * n - 1, vslot = ev % NSTAGE;
        mbar_wait(&kv_full[vslot], (ev / NSTAGE) & 1, p.dbg, SITE_MMA_V, ev);
        zero_v_tail(vslot, n - 1);
        wgmma_fence();
        issue_PV(o, pf, vslot, n > 1);
        wgmma_wait<0>();
        reg_fence(o);
        release(&kv_empty[vslot]);
      }
      ent += 2 * n;
    }

    // ---------------------------- epilogue ----------------------------
#pragma unroll
    for (int d = 1; d <= 2; d <<= 1) {
      l_lo += __shfl_xor_sync(0xffffffffu, l_lo, d);
      l_hi += __shfl_xor_sync(0xffffffffu, l_hi, d);
    }
    float inv_lo = (l_lo > 0.f) ? 1.0f / l_lo : 0.f;
    float inv_hi = (l_hi > 0.f) ? 1.0f / l_hi : 0.f;
    if constexpr (FP8 || DF8) {   // V = v_scale * V8: O = (P V8 / l) * v_scale; a split's partial too (the combine is linear)
      inv_lo *= p.v_scale;
      inv_hi *= p.v_scale;
    }
    // the sequence's row 0; packed layouts have sb = lse_sb = 0, dense ones q0 = 0
    const long long tile_off = p.ol.o(w.bidx, w.hidx, w.q0);
    if (p.lse != nullptr && tq == 0) {
      // a row that saw no key (l == 0) gets +inf; in a split-KV partial -inf, which tells the combine that the split
      // holds nothing for it
      const float none = p.nsplit > 1 ? -INFINITY : INFINITY;
      float* lrow = p.lse + w.split * p.lse_part_stride + p.ol.lse(w.bidx, w.hidx, w.q0);
      if (row_lo < S) lrow[row_lo] = l_lo > 0.f ? m_lo * p.scale + logf(l_lo) : none;
      if (row_hi < S) lrow[row_hi] = l_hi > 0.f ? m_hi * p.scale + logf(l_hi) : none;
    }

    if constexpr (OUT_F32) {
      // a split-KV partial without tiles is never read: its LSE = -inf gives it weight 0 in the combine
      const bool store = n > 0 || p.nsplit == 1;
      float* obase = p.out_f32 + w.split * p.part_stride + tile_off;
#pragma unroll
      for (int hr = 0; hr < 2; ++hr) {
        const int row = hr ? row_hi : row_lo;
        const float inv = hr ? inv_hi : inv_lo;
        if (store && row < S) {
          float* orow = obase + static_cast<long long>(row) * p.ol.ss + 2 * tq;
#pragma unroll
          for (int i = 0; i < D / 8; ++i)
            *reinterpret_cast<float2*>(orow + 8 * i) = make_float2(o[4 * i + 2 * hr] * inv, o[4 * i + 2 * hr + 1] * inv);
        }
      }
    } else {
      // registers -> swizzled staging (16-byte chunk c of row r sits at chunk (c & ~7) | ((c ^ r) & 7)) -> coalesced
      // 16-byte stores: consecutive threads write consecutive chunks of a row
      constexpr int ROW_BYTES = D * 2;
      constexpr int CHUNKS = ROW_BYTES / 16;
      uint8_t* stg = sStg + t * 64 * ROW_BYTES;
      const int rl = wq * 16 + g;                    // row inside this tile
#pragma unroll
      for (int i = 0; i < D / 8; ++i) {
        const int ph_lo = (i & ~7) | ((i ^ rl) & 7), ph_hi = (i & ~7) | ((i ^ (rl + 8)) & 7);
        *reinterpret_cast<uint32_t*>(stg + rl * ROW_BYTES + ph_lo * 16 + 4 * tq) =
            pack_16x2<IS_BF16>(o[4 * i + 0] * inv_lo, o[4 * i + 1] * inv_lo);
        *reinterpret_cast<uint32_t*>(stg + (rl + 8) * ROW_BYTES + ph_hi * 16 + 4 * tq) =
            pack_16x2<IS_BF16>(o[4 * i + 2] * inv_hi, o[4 * i + 3] * inv_hi);
      }
      named_bar_sync(1 + t, 128);
      uint8_t* obase = reinterpret_cast<uint8_t*>(p.out) + tile_off * 2;
      const int r128 = threadIdx.x & 127;
      const int trow0 = w.row0 + t * 64;
#pragma unroll 4
      for (int idx = r128; idx < 64 * CHUNKS; idx += 128) {
        const int rr = idx / CHUNKS, chunk = idx % CHUNKS;
        const int phys = (chunk & ~7) | ((chunk ^ rr) & 7);
        const uint4 v4 = *reinterpret_cast<const uint4*>(stg + rr * ROW_BYTES + phys * 16);
        const int rg = trow0 + rr;
        if (rg < S) {
          const long long off = static_cast<long long>(rg) * p.ol.ss * 2 + chunk * 16;
          st_global_v4(obase + off, v4);
          for (int d = 0; d < p.n_extra_dst; ++d)          // peer copies: posted stores over NVLink
            st_global_v4(reinterpret_cast<uint8_t*>(p.extra_dst[d]) + tile_off * 2 + off, v4);
        }
      }
      if (PERSIST) named_bar_sync(1 + t, 128);        // the staging is read out before the next item writes it
    }
  }
}

}  // namespace tfa
