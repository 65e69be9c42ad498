// tfa_rotary.cu -- instantiates and launches kvcache_rotary_append_kernel (fa_splitkv_combine.cuh) for tfa_api.cu.
//
// A translation unit of its own: the device compiler optimises a translation unit as one module, and instantiating
// the rotary kernels next to the forward changed the generated code of the KV-cache forward instantiations (same
// semantics, different SASS).  Kept apart, the forward's code is exactly what it was without rotary.
#include "../../include/tfa_b200.h"
#include "fa_splitkv_combine.cuh"

#include <cuda_runtime.h>

extern "C" void tfa_internal_count_launch(void);

namespace {

template <int D, bool IS_BF16>
void launch(const tfa::RotaryAppendParams& p, bool interleaved, int blocks, cudaStream_t stream) {
  auto kern = interleaved ? tfa::kvcache_rotary_append_kernel<D, IS_BF16, true>
                          : tfa::kvcache_rotary_append_kernel<D, IS_BF16, false>;
  kern<<<blocks, 256, 0, stream>>>(p);
}

}  // namespace

// One launch over q_chunks + ap.chunks 16-byte chunks, 256 per block; counted like every other launch.  Returns 0, a
// cudaError_t, or TFA_EINVAL_SHAPE when the grid does not fit.
int tfa_internal_launch_rotary_append(const tfa::RotaryAppendParams& p, int D, bool bf16, bool interleaved,
                                      cudaStream_t stream) {
  const long long blocks = (p.q_chunks + p.ap.chunks + 255) / 256;
  if (blocks > 0x7fffffffLL) return TFA_EINVAL_SHAPE;
  const int nb = static_cast<int>(blocks);
  if (D == 64) {
    if (bf16) launch<64, true>(p, interleaved, nb, stream);
    else launch<64, false>(p, interleaved, nb, stream);
  } else {
    if (bf16) launch<128, true>(p, interleaved, nb, stream);
    else launch<128, false>(p, interleaved, nb, stream);
  }
  tfa_internal_count_launch();
  return static_cast<int>(cudaGetLastError());
}
