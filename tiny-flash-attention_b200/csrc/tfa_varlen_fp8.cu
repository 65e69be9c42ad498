// tfa_varlen_fp8.cu -- instantiates the FP8 variable-length attention forward (kVarlenFp8 of fa_fwd_sm90.cuh: packed
// Q, K and V in e4m3 addressed through cu_seqlens, both products on 8-bit wgmma) and its launch (fa_fwd_launch.cuh,
// which declares this instantiation `extern template`): 2 head dims x causal x output dtype x fp32 output x 2 schedules
// = 32 kernels.
//
// A translation unit of its own, as tfa_fp8_fwd.cu, so that the existing instantiations are compiled exactly as they
// were without this mode.
#include "fa_fwd_launch.cuh"

template cudaError_t tfa::launch_forward<tfa::kVarlenFp8>(int D, bool causal, bool bf16, bool f32, const CUtensorMap& tq,
                                                          const CUtensorMap& tk, const CUtensorMap& tv,
                                                          const tfa::FwdParams& p, int nblocks, bool persist,
                                                          cudaStream_t stream);
