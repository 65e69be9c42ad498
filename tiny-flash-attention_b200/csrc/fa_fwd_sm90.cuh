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
// both at once, a packed variable-length batch of queries (cu_seqlens) against a (paged) KV cache.
#pragma once
#include "ptx_sm90.cuh"

namespace tfa {

enum : int { kDense = 0, kVarlen = 1, kCache = 2, kVarlenCache = 3 };

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
// LSE at element b*lse_sb + h*lse_sh + row of lse.  The host builds it once per call (tfa_api.cu); the combine and the
// empty-rows fill address out / lse through it, and set_output derives the forward's strides below from it.
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
  void* out;          // 16-bit output, element strides below
  // Fused exchange (multi-GPU): when n_extra_dst > 0 every 16-byte chunk of O is ALSO stored to these buffers
  // (same strides) -- peer GPUs' copies of the gathered output, mapped over NVLink.  Replaces the all-gather.
  void* extra_dst[7];
  int n_extra_dst;
  float* out_f32;     // fp32 output (validation build), same strides
  float* lse;         // (BH, S) fp32 or nullptr
  long long o_stride_b, o_stride_h, o_stride_s;  // elements
  int H;             // query heads
  int S;             // query rows
  int npairs;         // ceil(S / 128): Q-tile pairs per (batch, head)
  // Generalised problem (SURVEY.md 8f rows 2-3; reference: flash_attention_c/csrc/attn.cpp:121-124,182-183 for
  // Sq != Sk with a bottom-right aligned causal mask, csrc/archive_)/attn.cpp:61,375 for grouped K/V heads):
  int Sk;             // keys (== S for the reference's CuTe path)
  int causal_off;     // Sk - S >= 0: query row i sees keys j <= i + causal_off
  int kv_group;       // query heads per K/V head (1 = MHA)
  // split-KV: the grid carries nsplit work items per Q-tile pair, each covering split_tiles KV tiles and writing a
  // normalised fp32 partial O plus its LSE; tfa_splitkv_combine merges them.  nsplit == 1: split_tiles = all.
  int nsplit;
  int split_tiles;
  long long part_stride;      // out_f32 elements between consecutive splits
  long long lse_stride_bh;    // lse elements between consecutive (b,h)
  long long lse_part_stride;  // lse elements between consecutive splits
  // launch order (decode_work below): heads are taken in chunks of `head_chunk`; total (batch*head) count `BH`
  int head_chunk;
  int BH;
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

// watchdog call sites
enum : uint32_t { SITE_LOAD_EMPTY = 1, SITE_LOAD_Q = 2, SITE_MMA_Q = 3, SITE_MMA_K = 4, SITE_MMA_V = 5 };

constexpr float kRescaleThresholdLog2 = 8.0f;  // lazy rescale: tolerate P up to 2^8
// Register re-allocation after the prologue.  setmaxnreg moves registers inside the CTA's OWN pool, which is
// what the launch allocated: 384 threads x 168 = 64512.  2 softmax warpgroups x 240 + 1 producer warpgroup x 24
// = 504 x 128 = 64512.
constexpr uint32_t kRegsSoftmax = 240;
constexpr uint32_t kRegsProducer = 24;
static_assert((2 * kRegsSoftmax + kRegsProducer) * 128 <= 384 * 168, "setmaxnreg budget exceeds the CTA register pool");

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
// write.  The producer loads an item iff n > 0, the softmax warpgroups wait on its barriers iff n > 0: n > 0 implies
// live.
struct Item {
  int bh, bidx, hidx, hkv, split, jb, row0, n;
  int q0, k0, Sq, Sk, coff;
  bool live;
};
template <bool CAUSAL, int MODE>
__device__ __forceinline__ Item decode_item(int item, const FwdParams& p) {
  constexpr bool VARLEN = MODE == kVarlen;
  constexpr bool QPACK = MODE == kVarlen || MODE == kVarlenCache;    // packed queries: items past a sequence skipped
  Item w;
  int pr;
  decode_work(item, p.npairs, p.nsplit, p.head_chunk, p.BH, w.bh, w.split, pr);
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
  } else if constexpr (MODE == kCache) {
    w.q0 = 0;
    w.k0 = 0;
    w.Sq = p.S;
    w.Sk = cache_len(__ldg(p.cache_seqlens + w.bidx), p.capacity, p.snew) + p.snew;
    w.coff = w.Sk - w.Sq;           // may be negative, as for varlen
  } else if constexpr (MODE == kVarlenCache) {
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
  // causal: the item's last row sees keys <= last (none when last < 0, which only varlen and cache sequences can have)
  const int last = w.row0 + 127 + w.coff;
  const int nfull = CAUSAL ? ((MODE != kDense && last < 0) ? 0 : min(nkv_total, last / 128 + 1)) : nkv_total;
  w.n = max(0, min(nfull - w.jb, p.split_tiles));   // 0: a split-KV item wholly above the causal diagonal
  // dense: an item without tiles writes nothing (its rows belong to other splits); varlen: an item inside its sequence
  // always writes its rows, as O = 0 and LSE = +inf when they see no key (n == 0); cache: every item writes its rows,
  // a split without tiles too (LSE = -inf), so the combine can read every split's partial
  w.live = QPACK ? w.row0 < w.Sq : (MODE == kCache || w.n > 0);
  if (QPACK && !w.live) w.n = 0;     // past the sequence's end: the producer must skip it as the consumers do
  return w;
}

template <int D, bool CAUSAL, bool IS_BF16, bool OUT_F32, bool PERSIST, int MODE>
__global__ void __launch_bounds__(384, 1)
fa_fwd_sm90_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                   const __grid_constant__ CUtensorMap tmV, const FwdParams p) {
  constexpr bool QPACK = MODE == kVarlen || MODE == kVarlenCache;   // q / out / lse packed as varlen
  constexpr bool PAGED = MODE == kCache || MODE == kVarlenCache;    // K/V from a (paged) cache
  using C = FwdCfg<D>;
  constexpr int TILE = C::TILE_BYTES;
  constexpr int NSTAGE = C::NSTAGE;

  extern __shared__ uint8_t smem_raw[];
  // SWIZZLE_128B operands need 1024-byte alignment (the swizzle is a function of address bits 7..9)
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;                       // the item's two Q tiles: rows [0,64) tile 0, [64,128) tile 1
  uint8_t* sStg = smem + TILE;              // epilogue staging, 128 rows x D 16-bit
  uint8_t* sKV = smem + 2 * TILE;           // NSTAGE tiles
  uint64_t* bars = reinterpret_cast<uint64_t*>(sKV + NSTAGE * TILE);
  uint64_t* q_full = bars;
  uint64_t* q_empty = bars + 1;
  uint64_t* kv_full = bars + 2;             // [NSTAGE]
  uint64_t* kv_empty = kv_full + NSTAGE;    // [NSTAGE]

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
    for (int i = 0; i < NSTAGE; ++i) {
      mbar_init(&kv_full[i], 1);
      mbar_init(&kv_empty[i], 8);
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp < 4) {
    // =========================== TMA producer ===========================
    setmaxnreg_dec<kRegsProducer>();
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
            const uint32_t slot = ent % NSTAGE;
            mbar_wait(&kv_empty[slot], ((ent / NSTAGE) & 1) ^ 1, p.dbg, SITE_LOAD_EMPTY, ent);
            mbar_arrive_expect_tx(&kv_full[slot], TILE);
            const CUtensorMap* tm = kv ? &tmV : &tmK;
#pragma unroll
            for (int sl = 0; sl < C::SLABS; ++sl)
              tma_load_4d(sKV + slot * TILE + sl * C::SLAB_BYTES, tm, &kv_full[slot], sl * 64, ky, w.hkv, kw);
          }
        }
      }
    }
    return;
  }

  // ================= softmax / wgmma / epilogue warpgroup t =================
  setmaxnreg_inc<kRegsSoftmax>();
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
    auto issue_S = [&](float* s, uint32_t kslot) {
      const uint32_t k_addr = sKV_addr + kslot * TILE;
#pragma unroll
      for (int kk = 0; kk < D / 16; ++kk) {
        const uint32_t off = (kk / 4) * C::SLAB_BYTES + (kk % 4) * 32;
        MmaS::template ss<0>(s, gmma_desc(sQ_addr + off, 16, 1024), gmma_desc(k_addr + off, 16, 1024), kk > 0 ? 1u : 0u);
      }
      wgmma_commit();
    };
    // O += P V over 8 k-steps of 16 keys; V is MN-major: 16 key rows = 2048 B per k-step, LBO = next 64-column slab
    auto issue_PV = [&](float* o, const uint32_t* pf, uint32_t vslot, bool acc) {
      const uint32_t v_addr = sKV_addr + vslot * TILE;
#pragma unroll
      for (int kk = 0; kk < C::BN / 16; ++kk)
        MmaO::rs(o, pf + 4 * kk, gmma_desc(v_addr + kk * 2048, C::SLAB_BYTES, 1024), (acc || kk > 0) ? 1u : 0u);
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
    auto zero_v_tail = [&](uint32_t vslot, int jt) {
      if constexpr (PAGED) {
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
    uint32_t pf[32];         // P as the A operand: 8 k-steps x 4 registers of 16-bit pairs
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
    auto pack_P = [&]() {
#pragma unroll
      for (int kk = 0; kk < 8; ++kk) {
        pf[4 * kk + 0] = pack_16x2<IS_BF16>(s[8 * kk + 0], s[8 * kk + 1]);
        pf[4 * kk + 1] = pack_16x2<IS_BF16>(s[8 * kk + 2], s[8 * kk + 3]);
        pf[4 * kk + 2] = pack_16x2<IS_BF16>(s[8 * kk + 4], s[8 * kk + 5]);
        pf[4 * kk + 3] = pack_16x2<IS_BF16>(s[8 * kk + 6], s[8 * kk + 7]);
      }
    };

    // A varlen or cache item whose rows all see no key has no tiles: it waits on no barrier, its rows get O = 0 and
    // LSE = +inf (-inf for a split-KV partial).
    if (MODE == kDense || n > 0) {
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
    const float inv_lo = (l_lo > 0.f) ? 1.0f / l_lo : 0.f;
    const float inv_hi = (l_hi > 0.f) ? 1.0f / l_hi : 0.f;
    const long long tile_off =
        (QPACK ? static_cast<long long>(w.q0) * p.o_stride_s : static_cast<long long>(w.bidx) * p.o_stride_b) +
        static_cast<long long>(w.hidx) * p.o_stride_h;
    if (p.lse != nullptr && tq == 0) {
      if constexpr (QPACK) {
        // (H, total_q); a row that saw no key (l == 0) gets +inf.  Not for split-KV partials, whose -inf tells the
        // combine that the split holds nothing.
        float* lrow = p.lse + static_cast<long long>(w.hidx) * p.lse_stride_bh + w.q0;
        if (row_lo < S) lrow[row_lo] = l_lo > 0.f ? m_lo * p.scale + logf(l_lo) : INFINITY;
        if (row_hi < S) lrow[row_hi] = l_hi > 0.f ? m_hi * p.scale + logf(l_hi) : INFINITY;
      } else if constexpr (MODE == kCache) {
        // (B, H, S) as dense; a row that saw no key gets +inf, or -inf in a split-KV partial (as above)
        const float none = p.nsplit > 1 ? -INFINITY : INFINITY;
        float* lrow = p.lse + w.split * p.lse_part_stride + static_cast<long long>(w.bh) * p.lse_stride_bh;
        if (row_lo < S) lrow[row_lo] = l_lo > 0.f ? m_lo * p.scale + logf(l_lo) : none;
        if (row_hi < S) lrow[row_hi] = l_hi > 0.f ? m_hi * p.scale + logf(l_hi) : none;
      } else {
        float* lrow = p.lse + w.split * p.lse_part_stride + static_cast<long long>(w.bh) * p.lse_stride_bh;
        if (row_lo < S) lrow[row_lo] = m_lo * p.scale + logf(l_lo);
        if (row_hi < S) lrow[row_hi] = m_hi * p.scale + logf(l_hi);
      }
    }

    if constexpr (OUT_F32) {
      float* obase = p.out_f32 + w.split * p.part_stride + tile_off;
#pragma unroll
      for (int hr = 0; hr < 2; ++hr) {
        const int row = hr ? row_hi : row_lo;
        const float inv = hr ? inv_hi : inv_lo;
        if (row < S) {
          float* orow = obase + static_cast<long long>(row) * p.o_stride_s + 2 * tq;
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
          const long long off = static_cast<long long>(rg) * p.o_stride_s * 2 + chunk * 16;
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
