// fa_fwd_launch.cuh -- the host launch of one fa_fwd_sm90_kernel instantiation, shared by the forward translation
// units: the kernel of the chosen schedule, its shared-memory opt-in, the launch, and the causal x dtype x fp32
// dispatch.  The caller sizes the grid and counts the launch.
//
// tfa_varlen_kvcache.cu explicitly instantiates launch_forward<kVarlenCache>, tfa_kvcache_fp8.cu launch_forward<
// kCacheFp8> and launch_forward<kVarlenCacheFp8>, tfa_fp8_fwd.cu launch_forward<kDenseFp8> and tfa_varlen_fp8.cu
// launch_forward<kVarlenFp8>, and tfa_api.cu declares those instantiations `extern template`, so that each mode's 32
// kernels are compiled in that unit only (the comment there says why).
#pragma once
#include "fa_fwd_sm90.cuh"

#include <cuda.h>
#include <cuda_runtime.h>

namespace tfa {

template <int D, bool CAUSAL, bool IS_BF16, bool OUT_F32, int MODE>
cudaError_t launch_forward_inst(const CUtensorMap& tq, const CUtensorMap& tk, const CUtensorMap& tv, const FwdParams& p,
                                int nblocks, bool persist, cudaStream_t stream) {
  auto kern = persist ? fa_fwd_sm90_kernel<D, CAUSAL, IS_BF16, OUT_F32, true, MODE>
                      : fa_fwd_sm90_kernel<D, CAUSAL, IS_BF16, OUT_F32, false, MODE>;
  // cudaFuncSetAttribute is per device (context) and costs well under a microsecond: set it on every launch instead of
  // caching "done once" per process, which breaks the first launch on a second GPU of the same process.
  constexpr int smem = fwd_smem_bytes<D, MODE>();
  const cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  if (e != cudaSuccess) return e;
  kern<<<nblocks, FwdCfg<D>::THREADS, smem, stream>>>(tq, tk, tv, p);
  return cudaSuccess;
}

template <int D, int MODE>
cudaError_t launch_forward_d(bool causal, bool bf16, bool f32, const CUtensorMap& tq, const CUtensorMap& tk,
                             const CUtensorMap& tv, const FwdParams& p, int nblocks, bool persist, cudaStream_t s) {
#define TFA_GO(C_, B_, F_) return launch_forward_inst<D, C_, B_, F_, MODE>(tq, tk, tv, p, nblocks, persist, s)
  if (causal) {
    if (bf16) { if (f32) TFA_GO(true, true, true); else TFA_GO(true, true, false); }
    else      { if (f32) TFA_GO(true, false, true); else TFA_GO(true, false, false); }
  } else {
    if (bf16) { if (f32) TFA_GO(false, true, true); else TFA_GO(false, true, false); }
    else      { if (f32) TFA_GO(false, false, true); else TFA_GO(false, false, false); }
  }
#undef TFA_GO
}

// The forward of problem mode MODE over `nblocks` CTAs (the persistent kernel when `persist`), p.total_items work
// items.  Returns the shared-memory opt-in's error, or cudaSuccess once the kernel is enqueued: the caller reads the
// launch's own error (cudaGetLastError) when it counts the launch.
template <int MODE>
cudaError_t launch_forward(int D, bool causal, bool bf16, bool f32, const CUtensorMap& tq, const CUtensorMap& tk,
                           const CUtensorMap& tv, const FwdParams& p, int nblocks, bool persist, cudaStream_t stream) {
  if (D == 64) return launch_forward_d<64, MODE>(causal, bf16, f32, tq, tk, tv, p, nblocks, persist, stream);
  return launch_forward_d<128, MODE>(causal, bf16, f32, tq, tk, tv, p, nblocks, persist, stream);
}

}  // namespace tfa
