// fa_splitkv_combine.cuh -- the small HBM-bound kernel after the split-KV attention forward: splitkv_combine_kernel
// merges the per-split partial results,
//     O = sum_s exp(lse_s - LSE) * O_s ,  LSE = log sum_s exp(lse_s)
// -- the consumer of the row log-sum-exp the reference emits "for backward" and never uses
// (/root/reference/flash_attention_cutlass/csrc/flash_attention.cu:353,615-623,666-683).
//
// Every split writes the LSE of every row of its partial: a split that holds none of a row's keys (past its causal
// diagonal, or a row that sees no key at all) writes LSE = -inf, which gets weight 0 here, so its O is never loaded
// (the forward does not store the O of a split without tiles).  A row with no key in any split gets O = 0 and
// LSE = +inf, the convention of the reference's CuTe epilogue for an empty row (flash_attention.cu:620-623) and of the
// forward's single pass.
//
// A pure streaming kernel: one thread owns 4 consecutive head-dim elements of one row, a warp (D=128) or half-warp
// (D=64) owns a row, every global access is a full 16-byte (fp32 in) / 8-byte (16-bit out) vector.
// Roofline: HBM.  Algorithmic bytes per row: 4 nsplit + 4D (splits holding some of the row's keys) + 2D + 4.
//
// PACKED (the variable-length cache call): the partials are (nsplit, H, total_q, D), one row per packed query row of
// every head, each sequence's rows at their packed offsets; a row finds its sequence through packed_row_seq().
#pragma once
#include "ptx_sm90.cuh"
#include "fa_fwd_sm90.cuh"    // OutLayout, the forward's output addressing

namespace tfa {

// Packed query row r of a variable-length batch (cu = B + 1 offsets into total rows, each clamped to [0, total]):
// b = the sequence whose rows [cu[b], cu[b+1]) hold r, found by an upper-bound binary search over cu[0..B] that reads
// no other entry whatever cu holds (for non-monotonic offsets it still returns a b with cu[b] <= r < cu[b+1]), and
// i = r - cu[b].  True when r is one of the first min(Sq_b, S) rows of sequence b, the rows the forward computes.
__host__ __device__ __forceinline__ bool packed_row_seq(const int* cu, int B, int total, int S, int r, int& b, int& i) {
  int lo = 0, hi = B + 1;                      // the first k in [0, B] with clamp(cu[k]) > r, or B + 1
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (min(max(cu[mid], 0), total) <= r) lo = mid + 1; else hi = mid;
  }
  b = lo - 1;
  if (b < 0 || b >= B) return false;           // before the first offset, or at / past the last
  i = r - min(max(cu[b], 0), total);
  return i < S;
}

struct CombineParams {
  const float* o_part;        // [nsplit][rows][D] fp32, normalised partial outputs
  const float* lse_part;      // [nsplit][rows]
  void* out;                  // 16-bit (or fp32 when OUT_F32) output at `ol`
  float* lse;                 // or nullptr
  OutLayout ol;
  long long rows;             // B*H*S; PACKED: H*S, S = total_q
  int H, S;
  int nsplit;
  const int* cu_q;            // PACKED: the B + 1 sequence offsets, and max_seqlen_q rows per sequence
  int B, max_seqlen_q;
};

template <int D, bool IS_BF16, bool OUT_F32, bool PACKED = false>
__global__ void __launch_bounds__(256) splitkv_combine_kernel(const CombineParams p) {
  constexpr int TPR = D / 4;                   // threads per row
  constexpr int RPB = 256 / TPR;               // rows per block
  const int sub = threadIdx.x % TPR;
  const long long row = static_cast<long long>(blockIdx.x) * RPB + threadIdx.x / TPR;
  if (row >= p.rows) return;
  const int i = static_cast<int>(row % p.S);
  const long long bh = row / p.S;
  if constexpr (PACKED) {                      // i is the packed row, bh the head; ol.sb = ol.lse_sb = 0
    int seq, k;
    if (!packed_row_seq(p.cu_q, p.B, p.S, p.max_seqlen_q, i, seq, k)) return;
  }
  const long long part_rows = p.rows;
  float m = -INFINITY;
  for (int s = 0; s < p.nsplit; ++s) m = fmaxf(m, __ldg(p.lse_part + s * part_rows + row));
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  float wsum = 0.f;
  if (m > -INFINITY) {
    for (int s = 0; s < p.nsplit; ++s) {
      const float w = expf(__ldg(p.lse_part + s * part_rows + row) - m);    // 0 for a split without the row's keys
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

}  // namespace tfa
