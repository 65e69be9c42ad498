// tfa_selftest_fp8.cu -- bring-up kernel for the e4m3 wgmma primitives of the FP8 attention forward (kDenseFp8): the
// SS chain of S = Q K^T on 8-bit swizzled TMA tiles, and the RS chain of O += P V with P packed from the accumulator
// layout by pack_p_e4m3 and V^T written by the converter's vt_convert_unit, both in fp8_p_key order.  The host side
// (tests/test_fwd_fp8.py) checks the results against exact products.  A translation unit of its own, so that the
// 16-bit self tests are compiled as they were.
#include "../../include/tfa_b200.h"
#include "fa_fwd_sm90.cuh"

#include <cudaTypedefs.h>
#include <cuda_fp16.h>
#include <cuda_fp8.h>

extern "C" void tfa_internal_count_launch(void);
extern "C" void* tfa_internal_dbg_dev(void);
extern "C" void* tfa_internal_encode_fn(void);

namespace {
using namespace tfa;

struct Fp8TestParams {
  const uint8_t* a;     // mode 1: A (128 x 128 keys) read by threads
  const uint8_t* b;     // mode 1: (128 keys x N) row-major, read by threads
  float* c;             // in: the accumulator's starting value C0; out: C0 + chain * A B
  int chain;            // times the whole K-deep chain is issued into the one accumulator
  DebugRecord* dbg;
};

__device__ __forceinline__ float e4m3_to_f32(uint8_t x) {
  return __half2float(__half(__nv_cvt_fp8_to_halfraw(static_cast<__nv_fp8_storage_t>(x), __NV_E4M3)));
}

// C(128 x N) = C0 + chain x A(128 x K) * B as two m64 halves, one warpgroup: chain x K / 32 wgmma k-steps accumulate
// into one fp32 accumulator that starts at C0, as the forward's O does over a row's keys.  MODE 0: SS, A and B TMA-staged (K-byte rows).
// MODE 1: RS (K = 128), A packed in registers, B through the converter.
template <int N, int K, int MODE>
__global__ void __launch_bounds__(128, 1)
selftest_fp8_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                    const Fp8TestParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sA = smem;             // 128 x K bytes (mode 0)
  uint8_t* sB = smem + 16384;     // N x K bytes (mode 0) / V^T: N rows x 128 keys (mode 1)
  uint8_t* sRaw = smem + 32768;   // mode 1: 128 keys x N bytes
  uint64_t* bar = reinterpret_cast<uint64_t*>(smem + 49152);
  const int wq = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, tq = lane & 3;
  if constexpr (MODE == 0) {
    if (threadIdx.x == 0) {
      mbar_init(bar, 1);
      fence_mbar_init();
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      mbar_arrive_expect_tx(bar, 128 * K + N * K);
      tma_load_3d(sA, &tmA, bar, 0, 0, 0);
      tma_load_3d(sB, &tmB, bar, 0, 0, 0);
    }
    mbar_wait(bar, 0, p.dbg, 102, 0);
  } else {
    for (int i = threadIdx.x; i < 128 * N / 16; i += 128)
      reinterpret_cast<uint4*>(sRaw)[i] = reinterpret_cast<const uint4*>(p.b)[i];
    __syncthreads();
    for (int u = threadIdx.x; u < 2 * N; u += 128) vt_convert_unit<N>(smem_u32(sRaw), smem_u32(sB), u);
    fence_proxy_async_smem();
    __syncthreads();
  }

  for (int half = 0; half < 2; ++half) {
    float d[N / 2];
    const int row = half * 64 + wq * 16 + g;      // this thread's rows: row, row + 8
#pragma unroll
    for (int i = 0; i < N / 8; ++i) {
      d[4 * i] = p.c[row * N + 8 * i + 2 * tq];
      d[4 * i + 1] = p.c[row * N + 8 * i + 2 * tq + 1];
      d[4 * i + 2] = p.c[(row + 8) * N + 8 * i + 2 * tq];
      d[4 * i + 3] = p.c[(row + 8) * N + 8 * i + 2 * tq + 1];
    }
    uint32_t pf[16];
    if constexpr (MODE == 1) {
      float s[64];                                 // A as an accumulator: s[4i + 2h + e] = A[row + 8h][8i + 2tq + e]
#pragma unroll
      for (int i = 0; i < 16; ++i)
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int e = 0; e < 2; ++e) s[4 * i + 2 * h + e] = e4m3_to_f32(p.a[(row + 8 * h) * 128 + 8 * i + 2 * tq + e]);
      pack_p_e4m3(s, pf);
    }
    reg_fence(d);
    wgmma_fence();
    for (int rep = 0; rep < p.chain; ++rep) {
#pragma unroll
      for (int kk = 0; kk < K / 32; ++kk) {
        if constexpr (MODE == 0) {
          const uint32_t a_addr = smem_u32(sA) + half * 64 * K + kk * 32, b_addr = smem_u32(sB) + kk * 32;
          const uint64_t da = K == 128 ? gmma_desc(a_addr, 16, 1024) : gmma_desc_sw64(a_addr, 512);
          const uint64_t db = K == 128 ? gmma_desc(b_addr, 16, 1024) : gmma_desc_sw64(b_addr, 512);
          WgmmaE4m3<N>::ss(d, da, db, 1u);
        } else {
          WgmmaE4m3<N>::rs(d, pf + 4 * kk, gmma_desc(smem_u32(sB) + kk * 32, 16, 1024), 1u);
        }
      }
      wgmma_commit();
      wgmma_wait<0>();
      reg_fence(d);
      wgmma_fence();
    }
#pragma unroll
    for (int i = 0; i < N / 8; ++i) {
      p.c[row * N + 8 * i + 2 * tq] = d[4 * i];
      p.c[row * N + 8 * i + 2 * tq + 1] = d[4 * i + 1];
      p.c[(row + 8) * N + 8 * i + 2 * tq] = d[4 * i + 2];
      p.c[(row + 8) * N + 8 * i + 2 * tq + 1] = d[4 * i + 3];
    }
  }
}

// (rows x K) row-major e4m3 -> one box of all of it, swizzled to match its K-byte rows
int encode8(CUtensorMap* m, const void* base, uint64_t K, uint64_t rows) {
  auto encode = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(tfa_internal_encode_fn());
  if (!encode) return TFA_EDRIVER;
  const cuuint64_t dims[3] = {K, rows, 1};
  const cuuint64_t strides[2] = {K, K * rows};
  const cuuint32_t box[3] = {static_cast<cuuint32_t>(K), static_cast<cuuint32_t>(rows), 1};
  const cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = encode(m, CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, const_cast<void*>(base), dims, strides, box, estr,
                      CU_TENSOR_MAP_INTERLEAVE_NONE, K == 128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B,
                      CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : TFA_EDRIVER;
}

template <int N, int K, int MODE>
int launch(const CUtensorMap& tmA, const CUtensorMap& tmB, const Fp8TestParams& p, cudaStream_t stream) {
  const int smem = 49152 + 1024 + 64;
  auto kern = selftest_fp8_kernel<N, K, MODE>;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  if (e != cudaSuccess) return static_cast<int>(e);
  kern<<<1, 128, smem, stream>>>(tmA, tmB, p);
  tfa_internal_count_launch();
  return static_cast<int>(cudaGetLastError());
}

}  // namespace

extern "C" int tfa_selftest_wgmma_fp8(const void* a, const void* b, float* c, int N, int K, int mode, int chain,
                                      void* stream) {
  if (!a || !b || !c) return TFA_EINVAL_PTR;
  if (chain < 1 || chain > 4096) return TFA_EINVAL_SHAPE;
  if (mode == 0 ? (N != 128 || (K != 64 && K != 128)) : (mode != 1 || (N != 64 && N != 128) || K != 128))
    return TFA_EINVAL_DIM;
  Fp8TestParams p{static_cast<const uint8_t*>(a), static_cast<const uint8_t*>(b), c, chain,
                  static_cast<DebugRecord*>(tfa_internal_dbg_dev())};
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  CUtensorMap tmA{}, tmB{};
  if (mode == 0) {
    int rc;
    if ((rc = encode8(&tmA, a, K, 128)) || (rc = encode8(&tmB, b, K, N))) return rc;
    return K == 128 ? launch<128, 128, 0>(tmA, tmB, p, st) : launch<128, 64, 0>(tmA, tmB, p, st);
  }
  return N == 128 ? launch<128, 128, 1>(tmA, tmB, p, st) : launch<64, 128, 1>(tmA, tmB, p, st);
}
