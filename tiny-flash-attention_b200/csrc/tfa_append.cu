// tfa_append.cu -- instantiates and launches the KV-cache appends (kvcache_append_kernel and
// kvcache_rotary_append_kernel, fa_splitkv_combine.cuh) for tfa_api.cu.
//
// A translation unit of its own: the device compiler optimises a translation unit as one module, and instantiating
// the rotary kernels next to the forward changed the generated code of the KV-cache forward instantiations (same
// semantics, different SASS).  Kept apart, the forward's code is exactly what it was without the appends.
#include "../../include/tfa_b200.h"
#include "fa_splitkv_combine.cuh"

#include <cuda_runtime.h>

extern "C" void tfa_internal_count_launch(void);

namespace {

// One launch over `chunks` 16-byte chunks, 256 per block; counted like every other launch.
template <typename P>
int launch(void (*kern)(P), long long chunks, const P& p, cudaStream_t stream) {
  const long long blocks = (chunks + 255) / 256;
  if (blocks > 0x7fffffffLL) return TFA_EINVAL_SHAPE;
  kern<<<static_cast<int>(blocks), 256, 0, stream>>>(p);
  tfa_internal_count_launch();
  return static_cast<int>(cudaGetLastError());
}

template <int D, bool IS_BF16>
int launch_rotary(const tfa::RotaryAppendParams& p, bool interleaved, cudaStream_t stream) {
  return launch(interleaved ? tfa::kvcache_rotary_append_kernel<D, IS_BF16, true>
                            : tfa::kvcache_rotary_append_kernel<D, IS_BF16, false>,
                p.q_chunks + p.ap.chunks, p, stream);
}

}  // namespace

// The append of either cache call, over p.chunks chunks.  Returns 0, a cudaError_t, or TFA_EINVAL_SHAPE when the grid
// does not fit.
int tfa_internal_launch_append(const tfa::AppendParams& p, int D, cudaStream_t stream) {
  return launch(D == 64 ? tfa::kvcache_append_kernel<64> : tfa::kvcache_append_kernel<128>, p.chunks, p, stream);
}

// The rotary append, over q_chunks + ap.chunks chunks; returns as tfa_internal_launch_append.
int tfa_internal_launch_rotary_append(const tfa::RotaryAppendParams& p, int D, bool bf16, bool interleaved,
                                      cudaStream_t stream) {
  if (D == 64) return bf16 ? launch_rotary<64, true>(p, interleaved, stream)
                            : launch_rotary<64, false>(p, interleaved, stream);
  return bf16 ? launch_rotary<128, true>(p, interleaved, stream) : launch_rotary<128, false>(p, interleaved, stream);
}
