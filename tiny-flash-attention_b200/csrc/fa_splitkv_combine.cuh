// fa_splitkv_combine.cuh -- the small HBM-bound kernels either side of the attention forward when the problem
// is not the reference's square one (SURVEY.md 8f rows 2-3), plus the KV-cache append (kvcache_append_kernel, below):
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
  void* out;                  // 16-bit (or fp32 when OUT_F32) output, strided
  float* lse;                 // (B*H, lse_stride_bh) or nullptr
  long long o_stride_b, o_stride_h, o_stride_s;   // elements
  long long lse_stride_bh;
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
  const long long off = b * p.o_stride_b + h * p.o_stride_h + static_cast<long long>(i) * p.o_stride_s + sub * 4;
  if constexpr (OUT_F32) {
    *reinterpret_cast<float4*>(static_cast<float*>(p.out) + off) = acc;
  } else {
    uint2 v;
    v.x = pack_16x2<IS_BF16>(acc.x, acc.y);
    v.y = pack_16x2<IS_BF16>(acc.z, acc.w);
    *reinterpret_cast<uint2*>(static_cast<uint16_t*>(p.out) + off) = v;
  }
  if (p.lse != nullptr && sub == 0)
    p.lse[bh * p.lse_stride_bh + i] = wsum > 0.f ? m + logf(wsum) : INFINITY;
}

struct FillParams {
  void* out;
  float* lse;
  long long o_stride_b, o_stride_h, o_stride_s;
  long long lse_stride_bh;
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
  const long long off = b * p.o_stride_b + h * p.o_stride_h + static_cast<long long>(i) * p.o_stride_s + sub * 4;
  if constexpr (OUT_F32) *reinterpret_cast<float4*>(static_cast<float*>(p.out) + off) = make_float4(0.f, 0.f, 0.f, 0.f);
  else *reinterpret_cast<uint2*>(static_cast<uint16_t*>(p.out) + off) = make_uint2(0u, 0u);
  if (p.lse != nullptr && sub == 0) p.lse[bh * p.lse_stride_bh + i] = INFINITY;
}

// kvcache_append_kernel: writes k_new / v_new (B, snew, Hkv, D) into the (paged) KV cache at keys
// [L_b, L_b + snew) of each sequence, L_b = cache_len(cache_seqlens[b]), before the forward reads the cache.  One thread
// copies one 16-byte chunk of K and the same chunk of V.  cache_seqlens is not incremented.  A token whose block-table
// entry lies outside [0, num_blocks) is dropped: no store leaves the cache.  Algorithmic bytes: 2 * 2 * B*snew*Hkv*D
// read and written.
struct AppendParams {
  const void* k_new;
  const void* v_new;
  void* k_cache;
  void* v_cache;
  long long n_sb, n_ss, n_sh;     // element strides of k_new / v_new
  long long c_sb, c_ss, c_sh;     // element strides of the caches: block, row, head
  const int* cache_seqlens;
  const int* block_table;         // nullptr: contiguous cache
  long long bt_stride;
  int page, capacity, snew, num_blocks, Hkv;
  long long chunks;               // B * snew * Hkv * D / 8
};

template <int D>
__global__ void __launch_bounds__(256) kvcache_append_kernel(const AppendParams p) {
  constexpr int CPR = D / 8;                   // 16-byte chunks per row
  const long long c = static_cast<long long>(blockIdx.x) * 256 + threadIdx.x;
  if (c >= p.chunks) return;
  const int sub = static_cast<int>(c % CPR);
  long long r = c / CPR;
  const int h = static_cast<int>(r % p.Hkv);
  r /= p.Hkv;
  const int i = static_cast<int>(r % p.snew);
  const int b = static_cast<int>(r / p.snew);
  const long long dst = append_offset(p.cache_seqlens, p.block_table, p.bt_stride, b, i, h, p.page, p.capacity,
                                      p.snew, p.num_blocks, p.c_sb, p.c_ss, p.c_sh);
  if (dst < 0) return;
  const long long src = b * p.n_sb + i * p.n_ss + h * p.n_sh + sub * 8;
  const uint4 kx = __ldg(reinterpret_cast<const uint4*>(static_cast<const uint16_t*>(p.k_new) + src));
  const uint4 vx = __ldg(reinterpret_cast<const uint4*>(static_cast<const uint16_t*>(p.v_new) + src));
  *reinterpret_cast<uint4*>(static_cast<uint16_t*>(p.k_cache) + dst + sub * 8) = kx;
  *reinterpret_cast<uint4*>(static_cast<uint16_t*>(p.v_cache) + dst + sub * 8) = vx;
}

}  // namespace tfa
