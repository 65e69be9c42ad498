// tfa_kvcache_qkv8.cu -- instantiates the e4m3-query KV-cache forwards (kCacheQkv8, kVarlenCacheQkv8 of fa_fwd_sm90.cuh:
// e4m3 queries against the e4m3 cache, both products on 8-bit wgmma) and their launch (fa_fwd_launch.cuh, which declares
// these instantiations `extern template`): 2 modes x 2 head dims x causal x output dtype x fp32 output x 2 schedules =
// 64 kernels.
//
// A translation unit of its own, as tfa_kvcache_fp8.cu, so that the existing instantiations are compiled exactly as
// they were without these modes.
#include "fa_fwd_launch.cuh"

template cudaError_t tfa::launch_forward<tfa::kCacheQkv8>(int D, bool causal, bool bf16, bool f32, const CUtensorMap& tq,
                                                          const CUtensorMap& tk, const CUtensorMap& tv,
                                                          const tfa::FwdParams& p, int nblocks, bool persist,
                                                          cudaStream_t stream);
template cudaError_t tfa::launch_forward<tfa::kVarlenCacheQkv8>(int D, bool causal, bool bf16, bool f32,
                                                                const CUtensorMap& tq, const CUtensorMap& tk,
                                                                const CUtensorMap& tv, const tfa::FwdParams& p,
                                                                int nblocks, bool persist, cudaStream_t stream);
