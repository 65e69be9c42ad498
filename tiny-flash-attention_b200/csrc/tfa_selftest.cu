// tfa_selftest.cu -- bring-up kernels for the primitives the forward kernel is built from.
// One tiny CTA each; the host side (tests/test_umma_primitives.py) checks the raw results.
// They exist because descriptor conventions (swizzle, LBO/SBO, register fragment packing) cannot be
// verified without hardware, and a wrong guess inside the big kernel is much harder to localise.
#include "../../include/tfa_b200.h"
#include "ptx_sm90.cuh"

#include <cudaTypedefs.h>
#include <cstring>

extern "C" void tfa_internal_count_launch(void);
extern "C" void* tfa_internal_dbg_dev(void);
extern "C" void* tfa_internal_encode_fn(void);

namespace {
using namespace tfa;

__global__ void __launch_bounds__(128, 1)
selftest_tma_kernel(const __grid_constant__ CUtensorMap tm, int x0, int y0, int z0, uint4* dump, DebugRecord* dbg) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bar = reinterpret_cast<uint64_t*>(smem + 16384);
  if (threadIdx.x == 0) {
    mbar_init(bar, 1);
    fence_mbar_init();
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    mbar_arrive_expect_tx(bar, 16384);
    tma_load_3d(smem, &tm, bar, x0, y0, z0);
  }
  mbar_wait(bar, 0, dbg, 100, 0);
  for (int i = threadIdx.x; i < 1024; i += 128) dump[i] = reinterpret_cast<const uint4*>(smem)[i];
}

struct MmaTestParams {
  int N, K, mode;
  uint32_t lbo_b, sbo_b, kstep_b, slab_a, slab_b, flags;
  const uint16_t* a_gmem;   // mode 2: A read by threads
  float* c;
  DebugRecord* dbg;
};

// C(128 x N) = A(128 x K) * B as two m64 halves, one warpgroup.
// A: 128 x K.  smem A (modes 0,1): K/64 slabs of [128 rows x 128 B]; mode 2: registers, loaded from global.
// B mode 0: N x K K-major : K/64 slabs of [N rows x 128 B].
// B mode 1/2: K x N MN-major: N/64 slabs of [K rows x 128 B].
template <int N, bool IS_BF16>
__global__ void __launch_bounds__(128, 1)
selftest_mma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                    const MmaTestParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sA = smem;             // up to 32 KB
  uint8_t* sB = smem + 32768;     // up to 32 KB
  uint64_t* bar_ld = reinterpret_cast<uint64_t*>(smem + 65536);
  const int wq = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, tq = lane & 3;

  if (threadIdx.x == 0) {
    mbar_init(bar_ld, 1);
    fence_mbar_init();
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    const int nslab_b = (p.mode == 0) ? p.K / 64 : N / 64;
    const uint32_t bytes = (p.mode != 2 ? 128 * p.K * 2 : 0) + N * p.K * 2;
    mbar_arrive_expect_tx(bar_ld, bytes);
    if (p.mode != 2)
      for (int sl = 0; sl < p.K / 64; ++sl) tma_load_3d(sA + sl * p.slab_a, &tmA, bar_ld, sl * 64, 0, 0);
    for (int sl = 0; sl < nslab_b; ++sl) tma_load_3d(sB + sl * p.slab_b, &tmB, bar_ld, sl * 64, 0, 0);
  }
  mbar_wait(bar_ld, 0, p.dbg, 101, 0);

  const uint32_t a_addr = smem_u32(sA), b_addr = smem_u32(sB);
  for (int half = 0; half < 2; ++half) {
    float d[N / 2];
#pragma unroll
    for (int i = 0; i < N / 2; ++i) d[i] = 0.f;
    const int row = half * 64 + wq * 16 + g;      // this thread's rows: row, row + 8
    reg_fence(d);
    wgmma_fence();
    for (int k = 0; k < p.K / 16; ++k) {
      uint32_t b_off;
      if (p.mode == 0) b_off = (k / 4) * p.slab_b + (k % 4) * p.kstep_b;   // K-major B: 32 B per k-step inside a slab
      else b_off = k * p.kstep_b;                                          // MN-major B: 16 rows per k-step
      const uint64_t bd = gmma_desc(b_addr + b_off, p.lbo_b, p.sbo_b);
      if (p.mode == 2) {
        // A fragment: {row, cols 2tq..+1}, {row+8, same}, {row, cols 2tq+8..+9}, {row+8, same}, 16-bit pairs
        uint32_t a[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const int r = row + (q & 1) * 8, col = 16 * k + 2 * tq + (q >> 1) * 8;
          const uint32_t lo = p.a_gmem[r * p.K + col], hi = p.a_gmem[r * p.K + col + 1];
          a[q] = (p.flags & 1u) ? ((lo << 16) | hi) : ((hi << 16) | lo);
        }
        Wgmma<N, IS_BF16>::rs(d, a, bd, k > 0);
      } else {
        // A (K-major): 4 k-steps of 32 B inside a 128-B slab row, then the next slab; rows [64 half, +64)
        const uint32_t a_off = half * 64 * 128 + (k / 4) * p.slab_a + (k % 4) * 32;
        const uint64_t ad = gmma_desc(a_addr + a_off, 16, 1024);
        if (p.mode == 0) Wgmma<N, IS_BF16>::template ss<0>(d, ad, bd, k > 0);
        else Wgmma<N, IS_BF16>::template ss<1>(d, ad, bd, k > 0);
      }
    }
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(d);
#pragma unroll
    for (int i = 0; i < N / 8; ++i) {
      p.c[row * N + 8 * i + 2 * tq] = d[4 * i];
      p.c[row * N + 8 * i + 2 * tq + 1] = d[4 * i + 1];
      p.c[(row + 8) * N + 8 * i + 2 * tq] = d[4 * i + 2];
      p.c[(row + 8) * N + 8 * i + 2 * tq + 1] = d[4 * i + 3];
    }
  }
}

int encode2d(CUtensorMap* m, const void* base, int dtype, uint64_t inner, uint64_t rows, uint32_t box_rows) {
  auto encode = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(tfa_internal_encode_fn());
  if (!encode) return TFA_EDRIVER;
  const CUtensorMapDataType dt = (dtype == TFA_BF16) ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
  const cuuint64_t dims[3] = {inner, rows, 1};
  const cuuint64_t strides[2] = {inner * 2, inner * rows * 2};
  const cuuint32_t box[3] = {64, box_rows, 1};
  const cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = encode(m, dt, 3, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                      CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                      CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : TFA_EDRIVER;
}

}  // namespace

extern "C" {

int tfa_selftest_tma(const void* src, int D, int S, int BH, int x0, int y0, int z0, void* dump_16k, void* stream) {
  if (!src || !dump_16k) return TFA_EINVAL_PTR;
  auto encode = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(tfa_internal_encode_fn());
  if (!encode) return TFA_EDRIVER;
  CUtensorMap tm;
  const cuuint64_t dims[3] = {static_cast<cuuint64_t>(D), static_cast<cuuint64_t>(S), static_cast<cuuint64_t>(BH)};
  const cuuint64_t strides[2] = {static_cast<cuuint64_t>(D) * 2, static_cast<cuuint64_t>(D) * S * 2};
  const cuuint32_t box[3] = {64, 128, 1};
  const cuuint32_t estr[3] = {1, 1, 1};
  if (encode(&tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(src), dims, strides, box, estr,
             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
    return TFA_EDRIVER;
  const int smem = 16384 + 1024 + 64;
  selftest_tma_kernel<<<1, 128, smem, static_cast<cudaStream_t>(stream)>>>(
      tm, x0, y0, z0, static_cast<uint4*>(dump_16k), static_cast<DebugRecord*>(tfa_internal_dbg_dev()));
  tfa_internal_count_launch();
  return static_cast<int>(cudaGetLastError());
}

int tfa_selftest_umma(const void* a, const void* b, float* c, int N, int K, int mode, int dtype, const int* knobs,
                      void* stream) {
  if (!a || !b || !c) return TFA_EINVAL_PTR;
  if ((N != 64 && N != 128) || (K != 64 && K != 128)) return TFA_EINVAL_DIM;
  if (mode < 0 || mode > 2) return TFA_EINVAL_SHAPE;
  CUtensorMap tmA, tmB;
  int rc;
  if ((rc = encode2d(&tmA, a, dtype, K, 128, 128))) return rc;
  if (mode == 0) rc = encode2d(&tmB, b, dtype, K, N, N);   // (N x K), K contiguous
  else rc = encode2d(&tmB, b, dtype, N, K, K);             // (K x N), N contiguous
  if (rc) return rc;

  MmaTestParams p;
  std::memset(&p, 0, sizeof(p));
  p.N = N; p.K = K; p.mode = mode;
  p.slab_a = 128 * 128;
  if (mode == 0) { p.slab_b = N * 128; p.lbo_b = 16; p.sbo_b = 1024; p.kstep_b = 32; }
  else           { p.slab_b = K * 128; p.lbo_b = p.slab_b; p.sbo_b = 1024; p.kstep_b = 2048; }
  if (knobs) {
    if (knobs[0]) p.lbo_b = knobs[0];
    if (knobs[1]) p.sbo_b = knobs[1];
    if (knobs[2]) p.kstep_b = knobs[2];
    p.flags = knobs[3];
  }
  p.a_gmem = static_cast<const uint16_t*>(a);
  p.c = c;
  p.dbg = static_cast<DebugRecord*>(tfa_internal_dbg_dev());
  const int smem = 65536 + 1024 + 64;
  auto kern = (N == 64) ? (dtype == TFA_BF16 ? selftest_mma_kernel<64, true> : selftest_mma_kernel<64, false>)
                        : (dtype == TFA_BF16 ? selftest_mma_kernel<128, true> : selftest_mma_kernel<128, false>);
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  if (e != cudaSuccess) return static_cast<int>(e);
  kern<<<1, 128, smem, static_cast<cudaStream_t>(stream)>>>(tmA, tmB, p);
  tfa_internal_count_launch();
  return static_cast<int>(cudaGetLastError());
}

}  // extern "C"
