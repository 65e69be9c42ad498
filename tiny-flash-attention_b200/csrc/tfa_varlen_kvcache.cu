// tfa_varlen_kvcache.cu -- instantiates the kVarlenCache forward (fa_fwd_sm90.cuh) and its launch (fa_fwd_launch.cuh,
// which declares this instantiation `extern template`).
//
// A translation unit of its own, as tfa_append.cu: the device compiler optimises a translation unit as one module,
// and new kernels instantiated next to the forward can change the generated code of the existing instantiations.
// Kept apart, those are exactly what they were without this mode.
#include "fa_fwd_launch.cuh"

template cudaError_t tfa::launch_forward<tfa::kVarlenCache>(int D, bool causal, bool bf16, bool f32,
                                                            const CUtensorMap& tq, const CUtensorMap& tk,
                                                            const CUtensorMap& tv, const tfa::FwdParams& p, int nblocks,
                                                            bool persist, cudaStream_t stream);
