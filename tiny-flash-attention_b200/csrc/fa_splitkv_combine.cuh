// fa_splitkv_combine.cuh -- the small HBM-bound kernels either side of the attention forward when the problem
// is not the reference's square one (SURVEY.md 8f rows 2-3), plus the KV-cache append of both cache calls
// (kvcache_append_kernel, below), its rotary variant (kvcache_rotary_append_kernel) and their quantizing variants for
// an FP8 cache (kvcache_append_fp8_kernel, kvcache_rotary_append_fp8_kernel), all launched from tfa_append.cu:
//
//   * splitkv_combine_kernel: merges the per-split partial results of the split-KV forward,
//       O = sum_s exp(lse_s - LSE) * O_s ,  LSE = log sum_s exp(lse_s)
//     -- the consumer of the row log-sum-exp the reference emits "for backward" and never uses
//     (/root/reference/flash_attention_cutlass/csrc/flash_attention.cu:353,615-623,666-683);
//   * empty_rows_fill_kernel: causal with more queries than keys (bottom-right aligned mask,
//     /root/reference/flash_attention_c/csrc/attn.cpp:121-124): the first Sq-Sk query rows see no key at all.
//     They get O = 0 and LSE = +inf, the convention of the reference's CuTe epilogue for an empty row
//     (flash_attention.cu:620-623); the reference's CPU loop divides 0/0 there.
//
// Both are pure streaming kernels: one thread owns 4 consecutive head-dim elements of one row, a warp (D=128) or
// half-warp (D=64) owns a row, every global access is a full 16-byte (fp32 in) / 8-byte (16-bit out) vector.
// Roofline: HBM.  Algorithmic bytes per row: combine nsplit_valid*(4D+4) + 2D + 4, fill 2D + 4.
#pragma once
#include "ptx_sm90.cuh"
#include "fa_fwd_sm90.cuh"    // the KV-cache address helpers the append shares with the forward

namespace tfa {

struct CombineParams {
  const float* o_part;        // [nsplit][B*H*S][D] fp32, normalised partial outputs
  const float* lse_part;      // [nsplit][B*H*S]
  void* out;                  // 16-bit (or fp32 when OUT_F32) output at `ol`
  float* lse;                 // or nullptr
  OutLayout ol;
  long long rows;             // B*H*S
  int H, S;
  int nsplit, split_tiles;    // as launched
  int nkv_total;              // ceil(Sk / 128)
  int causal, causal_off;
};

template <int D, bool IS_BF16, bool OUT_F32>
__global__ void __launch_bounds__(256) splitkv_combine_kernel(const CombineParams p) {
  constexpr int TPR = D / 4;                   // threads per row
  constexpr int RPB = 256 / TPR;               // rows per block
  const int sub = threadIdx.x % TPR;
  const long long row = static_cast<long long>(blockIdx.x) * RPB + threadIdx.x / TPR;
  if (row >= p.rows) return;
  const int i = static_cast<int>(row % p.S);
  const long long bh = row / p.S;
  // which splits wrote this row: the forward skips a Q tile for splits entirely above its causal diagonal
  int nvalid = p.nsplit;
  if (p.causal) {
    const int tile_last = (i / 128) * 128 + 127;
    const int nfull = min(p.nkv_total, (tile_last + p.causal_off) / 128 + 1);
    nvalid = min(p.nsplit, (nfull + p.split_tiles - 1) / p.split_tiles);
  }
  const long long part_rows = p.rows;
  float m = -INFINITY;
  for (int s = 0; s < nvalid; ++s) m = fmaxf(m, __ldg(p.lse_part + s * part_rows + row));
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  float wsum = 0.f;
  if (m > -INFINITY) {
    for (int s = 0; s < nvalid; ++s) {
      const float w = expf(__ldg(p.lse_part + s * part_rows + row) - m);    // 0 for a fully masked partial
      if (w > 0.f) {
        const float4 o = __ldg(reinterpret_cast<const float4*>(p.o_part + (s * part_rows + row) * D) + sub);
        acc.x = fmaf(w, o.x, acc.x);
        acc.y = fmaf(w, o.y, acc.y);
        acc.z = fmaf(w, o.z, acc.z);
        acc.w = fmaf(w, o.w, acc.w);
        wsum += w;
      }
    }
  }
  const float inv = wsum > 0.f ? 1.0f / wsum : 0.f;
  acc.x *= inv; acc.y *= inv; acc.z *= inv; acc.w *= inv;
  const long long b = bh / p.H, h = bh % p.H;
  const long long off = p.ol.o(b, h, i) + sub * 4;
  if constexpr (OUT_F32) {
    *reinterpret_cast<float4*>(static_cast<float*>(p.out) + off) = acc;
  } else {
    uint2 v;
    v.x = pack_16x2<IS_BF16>(acc.x, acc.y);
    v.y = pack_16x2<IS_BF16>(acc.z, acc.w);
    *reinterpret_cast<uint2*>(static_cast<uint16_t*>(p.out) + off) = v;
  }
  if (p.lse != nullptr && sub == 0)
    p.lse[p.ol.lse(b, h, i)] = wsum > 0.f ? m + logf(wsum) : INFINITY;
}

struct FillParams {
  void* out;
  float* lse;
  OutLayout ol;
  long long rows;             // B*H*n_empty
  int H, n_empty;
};

template <int D, bool OUT_F32>
__global__ void __launch_bounds__(256) empty_rows_fill_kernel(const FillParams p) {
  constexpr int TPR = D / 4;
  constexpr int RPB = 256 / TPR;
  const int sub = threadIdx.x % TPR;
  const long long row = static_cast<long long>(blockIdx.x) * RPB + threadIdx.x / TPR;
  if (row >= p.rows) return;
  const int i = static_cast<int>(row % p.n_empty);
  const long long bh = row / p.n_empty;
  const long long b = bh / p.H, h = bh % p.H;
  const long long off = p.ol.o(b, h, i) + sub * 4;
  if constexpr (OUT_F32) *reinterpret_cast<float4*>(static_cast<float*>(p.out) + off) = make_float4(0.f, 0.f, 0.f, 0.f);
  else *reinterpret_cast<uint2*>(static_cast<uint16_t*>(p.out) + off) = make_uint2(0u, 0u);
  if (p.lse != nullptr && sub == 0) p.lse[p.ol.lse(b, h, i)] = INFINITY;
}

// kvcache_append_kernel: writes k_new / v_new into the (paged) KV cache at keys [L_b, L_b + n_b) of each sequence,
// before the forward reads the cache (L_b from cache_lens).  The dense-query call appends n_b = snew rows of
// (B, snew, Hkv, D) k_new / v_new.  The variable-length call (cu_q set) appends rows cu_q[b] + i, i < n_b =
// min(Sq_b, snew), of packed (total_q, Hkv, D) ones, with snew = max_seqlen_q as its forward's grid covers max_seqlen_q
// rows of every sequence: a chunk with i >= n_b returns, so no search over cu_seqlens is needed.  The grid is
// B * snew * Hkv * D/8 chunks; one thread copies one 16-byte chunk of K and the same chunk of V.  cache_seqlens is not
// incremented.  A token past the capacity or behind a block-table entry outside [0, num_blocks) is dropped: no store
// leaves the cache.  Algorithmic bytes: 2 * 2 * (appended tokens) * Hkv * D read and written.
struct AppendParams {
  const void* k_new;
  const void* v_new;
  void* k_cache;
  void* v_cache;
  long long n_sb, n_ss, n_sh;     // element strides of k_new / v_new (n_sb = 0 when packed)
  long long c_sb, c_ss, c_sh;     // element strides of the caches: block, row, head
  const int* cache_seqlens;
  const int* block_table;         // nullptr: contiguous cache
  long long bt_stride;
  const int* cu_q;                // nullptr: k_new / v_new are (B, snew, Hkv, D); else packed as q, total_q rows
  int total_q;
  int page, capacity, snew, num_blocks, Hkv;
  long long chunks;               // B * snew * Hkv * D / 8
};

// Chunk c < p.chunks of the append: 16-byte chunk `sub` of appended token i of sequence b at head h, read at element
// src of k_new / v_new and written at element dst of the caches, or dropped (dst < 0).
struct AppendChunk {
  int b, i, h, sub;
  long long src, dst;
};
template <int D>
__device__ __forceinline__ AppendChunk append_chunk(const AppendParams& p, long long c) {
  constexpr int CPR = D / 8;                   // 16-byte chunks per row
  AppendChunk a;
  a.sub = static_cast<int>(c % CPR);
  long long r = c / CPR;
  a.h = static_cast<int>(r % p.Hkv);
  r /= p.Hkv;
  a.i = static_cast<int>(r % p.snew);
  a.b = static_cast<int>(r / p.snew);
  int q0 = 0, n = p.snew;
  if (p.cu_q) {
    // the forward's clamps (decode_item): whatever cu_seqlens holds, no row outside [0, total_q) is read
    q0 = min(max(__ldg(p.cu_q + a.b), 0), p.total_q);
    const int q1 = min(max(__ldg(p.cu_q + a.b + 1), 0), p.total_q);
    n = min(max(q1 - q0, 0), p.snew);
  }
  a.dst = append_offset(__ldg(p.cache_seqlens + a.b), p.block_table, p.bt_stride, a.b, a.i, a.h, p.page, p.capacity, n,
                        p.num_blocks, p.c_sb, p.c_ss, p.c_sh);
  a.src = a.b * p.n_sb + (q0 + a.i) * p.n_ss + a.h * p.n_sh;
  return a;
}

template <int D>
__global__ void __launch_bounds__(256) kvcache_append_kernel(const AppendParams p) {
  const long long c = static_cast<long long>(blockIdx.x) * 256 + threadIdx.x;
  if (c >= p.chunks) return;
  const AppendChunk a = append_chunk<D>(p, c);
  if (a.dst < 0) return;
  const long long src = a.src + a.sub * 8;
  const uint4 kx = __ldg(reinterpret_cast<const uint4*>(static_cast<const uint16_t*>(p.k_new) + src));
  const uint4 vx = __ldg(reinterpret_cast<const uint4*>(static_cast<const uint16_t*>(p.v_new) + src));
  *reinterpret_cast<uint4*>(static_cast<uint16_t*>(p.k_cache) + a.dst + a.sub * 8) = kx;
  *reinterpret_cast<uint4*>(static_cast<uint16_t*>(p.v_cache) + a.dst + a.sub * 8) = vx;
}

// ---- rotary position embedding (RoPE) for the KV-cache forward: flash-attn's rotary_cos / rotary_sin ----
// The table position of query or appended key i of a sequence with clamped cached length cache_len: appended keys sit
// at cache_len + i; query rows too when causal, every query row at cache_len otherwise.  Clamped to seqlen_ro - 1 so
// that no cos/sin read leaves the table; only a query row can get there (Sq > Snew near the capacity), since a key
// position is below capacity <= seqlen_ro.
__host__ __device__ __forceinline__ int rotary_pos(int cache_len, int i, bool causal, bool is_query, int seqlen_ro) {
  const int pos = (is_query && !causal) ? cache_len : cache_len + i;
  return min(pos, seqlen_ro - 1);
}

// fp32 arithmetic with one IEEE rounding each, written as PTX so that nvcc can neither contract a product and a sum
// into an FMA nor flush denormals (the build uses --use_fast_math): the rotation is then bit-identical to the same
// formula evaluated by eager torch in fp32.
__device__ __forceinline__ float mul_rn(float a, float b) {
  float d;
  asm("mul.rn.f32 %0, %1, %2;" : "=f"(d) : "f"(a), "f"(b));
  return d;
}
__device__ __forceinline__ float add_rn(float a, float b) {
  float d;
  asm("add.rn.f32 %0, %1, %2;" : "=f"(d) : "f"(a), "f"(b));
  return d;
}
__device__ __forceinline__ float sub_rn(float a, float b) {
  float d;
  asm("sub.rn.f32 %0, %1, %2;" : "=f"(d) : "f"(a), "f"(b));
  return d;
}
// element t (0..7) of a 16-byte chunk of 16-bit values, widened exactly to fp32
template <bool IS_BF16>
__device__ __forceinline__ float widen16(const uint4& v, int t) {
  const uint32_t w = (&v.x)[t >> 1];
  const uint32_t bits = (t & 1) ? (w >> 16) : (w & 0xffffu);
  if constexpr (IS_BF16) return __uint_as_float(bits << 16);
  float f;
  asm("cvt.f32.f16 %0, %1;" : "=f"(f) : "h"(static_cast<unsigned short>(bits)));
  return f;
}

// Chunk `sub` (elements [8 sub, 8 sub + 8)) of `row` rotated by the cos/sin table row `cs_row` (rotary_dim / 2
// entries each).  Each pair (x0, x1) becomes x0' = x0 c - x1 s, x1' = x0 s + x1 c in fp32, rounded once to 16 bits.
// Pairs are (j, j + rotary_dim/2) with angle j (GPT-NeoX), or (2j, 2j+1) with angle j when INTERLEAVED (GPT-J).
// Elements [rotary_dim, D) pass through.  rotary_dim is a multiple of 16, so a chunk is all rotated or all passed, and
// the NeoX partner of a chunk is another whole chunk.
template <bool IS_BF16, bool INTERLEAVED>
__device__ __forceinline__ uint4 rotate_chunk(const uint16_t* row, int sub, const uint16_t* cos_row,
                                              const uint16_t* sin_row, int rotary_dim) {
  const uint4 x = __ldg(reinterpret_cast<const uint4*>(row) + sub);
  const int e0 = sub * 8;
  if (e0 >= rotary_dim) return x;
  float r[8];
  if constexpr (INTERLEAVED) {
    const uint2 c2 = __ldg(reinterpret_cast<const uint2*>(cos_row + e0 / 2));
    const uint2 s2 = __ldg(reinterpret_cast<const uint2*>(sin_row + e0 / 2));
    const uint4 c = make_uint4(c2.x, c2.y, 0u, 0u), s = make_uint4(s2.x, s2.y, 0u, 0u);
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      const float x0 = widen16<IS_BF16>(x, 2 * t), x1 = widen16<IS_BF16>(x, 2 * t + 1);
      const float ct = widen16<IS_BF16>(c, t), st = widen16<IS_BF16>(s, t);
      r[2 * t] = sub_rn(mul_rn(x0, ct), mul_rn(x1, st));
      r[2 * t + 1] = add_rn(mul_rn(x0, st), mul_rn(x1, ct));
    }
  } else {
    const int half = rotary_dim / 2;
    const bool first = e0 < half;
    const int j0 = first ? e0 : e0 - half;                       // angle of element 0 of this chunk
    const uint4 y = __ldg(reinterpret_cast<const uint4*>(row + (first ? e0 + half : e0 - half)));   // the partners
    const uint4 c = __ldg(reinterpret_cast<const uint4*>(cos_row + j0));
    const uint4 s = __ldg(reinterpret_cast<const uint4*>(sin_row + j0));
#pragma unroll
    for (int t = 0; t < 8; ++t) {
      const float xt = widen16<IS_BF16>(x, t), yt = widen16<IS_BF16>(y, t);
      const float ct = widen16<IS_BF16>(c, t), st = widen16<IS_BF16>(s, t);
      r[t] = first ? sub_rn(mul_rn(xt, ct), mul_rn(yt, st))      // x0' = x0 c - x1 s  (x0 = x, x1 = y)
                   : add_rn(mul_rn(yt, st), mul_rn(xt, ct));     // x1' = x0 s + x1 c  (x0 = y, x1 = x)
    }
  }
  return make_uint4(pack_16x2<IS_BF16>(r[0], r[1]), pack_16x2<IS_BF16>(r[2], r[3]), pack_16x2<IS_BF16>(r[4], r[5]),
                    pack_16x2<IS_BF16>(r[6], r[7]));
}

// kvcache_rotary_append_kernel: the append of kvcache_append_kernel with RoPE, plus the rotated queries, in one launch
// (the dense-query call only: cu_q is nullptr).  Chunks [0, q_chunks) write rot(q) into the contiguous (B, Sq, Hq, D)
// buffer q_rot, which the forward then reads in place of q; the remaining chunks write rot(k_new) and v_new
// (unrotated) into the cache at keys [L_b, L_b + snew), through the plain append's append_chunk().  Positions:
// rotary_pos().  One thread per 16-byte output chunk (a NeoX chunk also reads its partner chunk and 16 bytes each of
// cos and sin).  Algorithmic bytes: 2 * B*Sq*Hq*D * 2 (q in, q_rot out) + 2 * 2 * B*snew*Hkv*D * 2 (k/v in and out),
// plus the cos/sin rows.
struct RotaryAppendParams {
  AppendParams ap;                // the append; ap.chunks = B * snew * Hkv * D / 8
  const void* q;
  void* q_rot;                    // (B, Sq, Hq, D) contiguous
  long long q_sb, q_ss, q_sh;     // element strides of q
  const void* cos;                // (seqlen_ro, rotary_dim / 2) contiguous, q's dtype
  const void* sin;
  int Sq, Hq, rotary_dim, seqlen_ro, causal;
  long long q_chunks;             // B * Sq * Hq * D / 8
};

// The two halves of kvcache_rotary_append_kernel (below) as functions, for its FP8 variant.  The 16-bit kernel keeps
// its own copy of the body: built from these functions, its interleaved instantiations compile to different SASS (8
// more instructions at D = 128), and its generated code is kept as it was.
// Chunk c < q_chunks of the rotary append: rot(q) into q_rot.
template <int D, bool IS_BF16, bool INTERLEAVED>
__device__ __forceinline__ void rotary_q_chunk(const RotaryAppendParams& p, long long c) {
  constexpr int CPR = D / 8;                   // 16-byte chunks per row
  const AppendParams& a = p.ap;
  const uint16_t* cos_tab = static_cast<const uint16_t*>(p.cos);
  const uint16_t* sin_tab = static_cast<const uint16_t*>(p.sin);
  const int sub = static_cast<int>(c % CPR);
  long long r = c / CPR;                       // row index over (B, Sq, Hq), Hq fastest
  const int h = static_cast<int>(r % p.Hq);
  r /= p.Hq;
  const int i = static_cast<int>(r % p.Sq);
  const int b = static_cast<int>(r / p.Sq);
  const int len = cache_len(__ldg(a.cache_seqlens + b), a.capacity, a.snew);
  const long long ro =
      static_cast<long long>(rotary_pos(len, i, p.causal != 0, true, p.seqlen_ro)) * (p.rotary_dim / 2);
  const uint16_t* row = static_cast<const uint16_t*>(p.q) + b * p.q_sb + i * p.q_ss + h * p.q_sh;
  const uint4 y = rotate_chunk<IS_BF16, INTERLEAVED>(row, sub, cos_tab + ro, sin_tab + ro, p.rotary_dim);
  reinterpret_cast<uint4*>(static_cast<uint16_t*>(p.q_rot) + ((static_cast<long long>(b) * p.Sq + i) * p.Hq + h) * D)
      [sub] = y;
}
// The key half: rot(k_new) and v_new of appended chunk k (k.dst >= 0), as 16-bit chunks.
template <bool IS_BF16, bool INTERLEAVED>
__device__ __forceinline__ void rotary_kv_chunk(const RotaryAppendParams& p, const AppendChunk& k, uint4& kx,
                                                uint4& vx) {
  const AppendParams& a = p.ap;
  const int len = cache_len(__ldg(a.cache_seqlens + k.b), a.capacity, a.snew);
  const long long ro =
      static_cast<long long>(rotary_pos(len, k.i, p.causal != 0, false, p.seqlen_ro)) * (p.rotary_dim / 2);
  kx = rotate_chunk<IS_BF16, INTERLEAVED>(static_cast<const uint16_t*>(a.k_new) + k.src, k.sub,
                                          static_cast<const uint16_t*>(p.cos) + ro,
                                          static_cast<const uint16_t*>(p.sin) + ro, p.rotary_dim);
  vx = __ldg(reinterpret_cast<const uint4*>(static_cast<const uint16_t*>(a.v_new) + k.src) + k.sub);
}

template <int D, bool IS_BF16, bool INTERLEAVED>
__global__ void __launch_bounds__(256) kvcache_rotary_append_kernel(const RotaryAppendParams p) {
  constexpr int CPR = D / 8;                   // 16-byte chunks per row
  const long long c = static_cast<long long>(blockIdx.x) * 256 + threadIdx.x;
  const AppendParams& a = p.ap;
  const uint16_t* cos_tab = static_cast<const uint16_t*>(p.cos);
  const uint16_t* sin_tab = static_cast<const uint16_t*>(p.sin);
  if (c < p.q_chunks) {
    const int sub = static_cast<int>(c % CPR);
    long long r = c / CPR;                     // row index over (B, Sq, Hq), Hq fastest
    const int h = static_cast<int>(r % p.Hq);
    r /= p.Hq;
    const int i = static_cast<int>(r % p.Sq);
    const int b = static_cast<int>(r / p.Sq);
    const int len = cache_len(__ldg(a.cache_seqlens + b), a.capacity, a.snew);
    const long long ro =
        static_cast<long long>(rotary_pos(len, i, p.causal != 0, true, p.seqlen_ro)) * (p.rotary_dim / 2);
    const uint16_t* row = static_cast<const uint16_t*>(p.q) + b * p.q_sb + i * p.q_ss + h * p.q_sh;
    const uint4 y = rotate_chunk<IS_BF16, INTERLEAVED>(row, sub, cos_tab + ro, sin_tab + ro, p.rotary_dim);
    reinterpret_cast<uint4*>(static_cast<uint16_t*>(p.q_rot) + ((static_cast<long long>(b) * p.Sq + i) * p.Hq + h) * D)
        [sub] = y;
    return;
  }
  if (c - p.q_chunks >= a.chunks) return;
  const AppendChunk k = append_chunk<D>(a, c - p.q_chunks);
  if (k.dst < 0) return;
  const int len = cache_len(__ldg(a.cache_seqlens + k.b), a.capacity, a.snew);
  const long long ro =
      static_cast<long long>(rotary_pos(len, k.i, p.causal != 0, false, p.seqlen_ro)) * (p.rotary_dim / 2);
  const uint4 kx = rotate_chunk<IS_BF16, INTERLEAVED>(static_cast<const uint16_t*>(a.k_new) + k.src, k.sub,
                                                      cos_tab + ro, sin_tab + ro, p.rotary_dim);
  const uint4 vx = __ldg(reinterpret_cast<const uint4*>(static_cast<const uint16_t*>(a.v_new) + k.src) + k.sub);
  *reinterpret_cast<uint4*>(static_cast<uint16_t*>(a.k_cache) + k.dst + k.sub * 8) = kx;
  *reinterpret_cast<uint4*>(static_cast<uint16_t*>(a.v_cache) + k.dst + k.sub * 8) = vx;
}

// ---- FP8 (e4m3) cache: the appends quantize what they would have stored ----
// A stored key is K8 = e4m3_rn_satfinite(k / k_scale), a value V8 = e4m3_rn_satfinite(v / v_scale): an IEEE fp32
// division (div.rn, not the fast-math approximation the build would otherwise emit), rounded to nearest-even and
// saturated to +-448 -- bit-identical to torch's (x.float() / scale).clamp(-448, 448).to(torch.float8_e4m3fn).  With
// rotary the key is rotated and rounded to q's dtype first, as the 16-bit rotary append stores it.
struct KvQuant {
  float k_scale, v_scale;
};
__device__ __forceinline__ float div_rn(float a, float b) {
  float d;
  asm("div.rn.f32 %0, %1, %2;" : "=f"(d) : "f"(a), "f"(b));
  return d;
}
// 8 16-bit values -> 8 e4m3 codes, element 0 in the low byte
template <bool IS_BF16>
__device__ __forceinline__ uint2 quantize_chunk(const uint4& x, float scale) {
  uint32_t w[2];
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    unsigned short lo, hi;
    asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;"
        : "=h"(lo)
        : "f"(div_rn(widen16<IS_BF16>(x, 4 * i + 1), scale)), "f"(div_rn(widen16<IS_BF16>(x, 4 * i), scale)));
    asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;"
        : "=h"(hi)
        : "f"(div_rn(widen16<IS_BF16>(x, 4 * i + 3), scale)), "f"(div_rn(widen16<IS_BF16>(x, 4 * i + 2), scale)));
    w[i] = static_cast<uint32_t>(lo) | (static_cast<uint32_t>(hi) << 16);
  }
  return make_uint2(w[0], w[1]);
}

// kvcache_append_kernel into an e4m3 cache: 16 bytes of k_new / v_new in, 8 bytes of codes out per thread.
template <int D, bool IS_BF16>
__global__ void __launch_bounds__(256) kvcache_append_fp8_kernel(const AppendParams p, const KvQuant qs) {
  const long long c = static_cast<long long>(blockIdx.x) * 256 + threadIdx.x;
  if (c >= p.chunks) return;
  const AppendChunk a = append_chunk<D>(p, c);
  if (a.dst < 0) return;
  const long long src = a.src + a.sub * 8;
  const uint4 kx = __ldg(reinterpret_cast<const uint4*>(static_cast<const uint16_t*>(p.k_new) + src));
  const uint4 vx = __ldg(reinterpret_cast<const uint4*>(static_cast<const uint16_t*>(p.v_new) + src));
  *reinterpret_cast<uint2*>(static_cast<uint8_t*>(p.k_cache) + a.dst + a.sub * 8) = quantize_chunk<IS_BF16>(kx, qs.k_scale);
  *reinterpret_cast<uint2*>(static_cast<uint8_t*>(p.v_cache) + a.dst + a.sub * 8) = quantize_chunk<IS_BF16>(vx, qs.v_scale);
}

// kvcache_rotary_append_kernel into an e4m3 cache: rot(q) to q_rot as there, rot(k_new) and v_new quantized.
template <int D, bool IS_BF16, bool INTERLEAVED>
__global__ void __launch_bounds__(256) kvcache_rotary_append_fp8_kernel(const RotaryAppendParams p, const KvQuant qs) {
  const long long c = static_cast<long long>(blockIdx.x) * 256 + threadIdx.x;
  const AppendParams& a = p.ap;
  if (c < p.q_chunks) {
    rotary_q_chunk<D, IS_BF16, INTERLEAVED>(p, c);
    return;
  }
  if (c - p.q_chunks >= a.chunks) return;
  const AppendChunk k = append_chunk<D>(a, c - p.q_chunks);
  if (k.dst < 0) return;
  uint4 kx, vx;
  rotary_kv_chunk<IS_BF16, INTERLEAVED>(p, k, kx, vx);
  *reinterpret_cast<uint2*>(static_cast<uint8_t*>(a.k_cache) + k.dst + k.sub * 8) = quantize_chunk<IS_BF16>(kx, qs.k_scale);
  *reinterpret_cast<uint2*>(static_cast<uint8_t*>(a.v_cache) + k.dst + k.sub * 8) = quantize_chunk<IS_BF16>(vx, qs.v_scale);
}

}  // namespace tfa
