// tfa_append.cu -- instantiates and launches the KV-cache append (kvcache_append_kernel, fa_kvcache_append.cuh) for
// tfa_api.cu.
//
// A translation unit of its own: the device compiler optimises a translation unit as one module, and instantiating
// the rotary appends next to the forward changed the generated code of the KV-cache forward instantiations (same
// semantics, different SASS).  Kept apart, the forward's code is exactly what it was without the appends.
#include "../../include/tfa_b200.h"
#include "fa_kvcache_append.cuh"

#include <cuda_runtime.h>

extern "C" void tfa_internal_count_launch(void);

namespace {

using tfa::AppendKernelParams;
using tfa::KvQuant;
using tfa::kvcache_append_kernel;

// One launch over `chunks` 16-byte chunks, 256 per block, with the kernel's arguments `args`; counted like every other
// launch.
template <typename... P>
int launch(void (*kern)(P...), long long chunks, cudaStream_t stream, const P&... args) {
  const long long blocks = (chunks + 255) / 256;
  if (blocks > 0x7fffffffLL) return TFA_EINVAL_SHAPE;
  kern<<<static_cast<int>(blocks), 256, 0, stream>>>(args...);
  tfa_internal_count_launch();
  return static_cast<int>(cudaGetLastError());
}

// The dtype and cache-type dispatch of one head dimension and rotary layout.  The 16-bit append without rotary copies
// bits, so one instantiation serves both dtypes.  `q8`: q is quantized too (FP8 cache only).
template <int D, bool ROTARY, bool INTERLEAVED>
int launch_append(const AppendKernelParams& p, const KvQuant* qs, bool q8, bool bf16, cudaStream_t stream) {
  const long long chunks = p.q_chunks + p.ap.chunks;
  if (q8)
    return launch(bf16 ? kvcache_append_kernel<D, true, ROTARY, INTERLEAVED, true, true>
                       : kvcache_append_kernel<D, false, ROTARY, INTERLEAVED, true, true>,
                  chunks, stream, p, *qs);
  if (qs)
    return launch(bf16 ? kvcache_append_kernel<D, true, ROTARY, INTERLEAVED, true>
                       : kvcache_append_kernel<D, false, ROTARY, INTERLEAVED, true>,
                  chunks, stream, p, *qs);
  if constexpr (!ROTARY)
    return launch(kvcache_append_kernel<D, false, false, false, false>, chunks, stream, p, KvQuant{});
  else
    return launch(bf16 ? kvcache_append_kernel<D, true, true, INTERLEAVED, false>
                       : kvcache_append_kernel<D, false, true, INTERLEAVED, false>,
                  chunks, stream, p, KvQuant{});
}

template <int D>
int launch_append(const AppendKernelParams& p, const KvQuant* qs, bool q8, bool bf16, bool rotary, bool interleaved,
                  cudaStream_t stream) {
  if (!rotary) return launch_append<D, false, false>(p, qs, q8, bf16, stream);
  return interleaved ? launch_append<D, true, true>(p, qs, q8, bf16, stream)
                     : launch_append<D, true, false>(p, qs, q8, bf16, stream);
}

}  // namespace

// The append of either cache call, over p.q_chunks + p.ap.chunks chunks.  `qs` nullptr: a 16-bit cache; otherwise an
// FP8 (e4m3) one, into which k_new / v_new (rot(k_new) with rotary) are quantized with its scales.  `q8` (with `qs`):
// the query chunks write q (rot(q) with rotary) quantized with qs->q_scale into the e4m3 scratch p.q_rot.  `rotary`: q
// and k_new are rotated, with (2j, 2j+1) pairs when `interleaved`.  Returns 0, a cudaError_t, or TFA_EINVAL_SHAPE when
// the grid does not fit.
int tfa_internal_launch_append(const AppendKernelParams& p, const KvQuant* qs, bool q8, int D, bool bf16, bool rotary,
                               bool interleaved, cudaStream_t stream) {
  return D == 64 ? launch_append<64>(p, qs, q8, bf16, rotary, interleaved, stream)
                 : launch_append<128>(p, qs, q8, bf16, rotary, interleaved, stream);
}
