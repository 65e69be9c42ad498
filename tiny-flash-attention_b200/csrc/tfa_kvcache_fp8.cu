// tfa_kvcache_fp8.cu -- instantiates the FP8-cache forwards (kCacheFp8, kVarlenCacheFp8 of fa_fwd_sm90.cuh) and their
// launch (fa_fwd_launch.cuh, which declares these instantiations `extern template`).
//
// A translation unit of its own, as tfa_varlen_kvcache.cu: the device compiler optimises a translation unit as one
// module, and new kernels instantiated next to the forward can change the generated code of the existing
// instantiations.  Kept apart, those are exactly what they were without these modes.
#include "fa_fwd_launch.cuh"

template cudaError_t tfa::launch_forward<tfa::kCacheFp8>(int D, bool causal, bool bf16, bool f32, const CUtensorMap& tq,
                                                         const CUtensorMap& tk, const CUtensorMap& tv,
                                                         const tfa::FwdParams& p, int nblocks, bool persist,
                                                         cudaStream_t stream);
template cudaError_t tfa::launch_forward<tfa::kVarlenCacheFp8>(int D, bool causal, bool bf16, bool f32,
                                                               const CUtensorMap& tq, const CUtensorMap& tk,
                                                               const CUtensorMap& tv, const tfa::FwdParams& p,
                                                               int nblocks, bool persist, cudaStream_t stream);
