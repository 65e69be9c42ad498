// tfa_varlen_kvcache.cu -- instantiates and launches the kVarlenCache forward (fa_fwd_sm90.cuh) and its append
// (kvcache_varlen_append_kernel, fa_splitkv_combine.cuh) for tfa_api.cu, and exports their address helpers for the
// CPU tests.
//
// A translation unit of its own, as tfa_rotary.cu: the device compiler optimises a translation unit as one module,
// and new kernels instantiated next to the forward can change the generated code of the existing instantiations.
// Kept apart, those are exactly what they were without this mode.  This is the only place the mode's kernels are
// instantiated: launch_fwd in tfa_api.cu must never reach its own dispatch for kVarlenCache (see the comment there).
#include "../../include/tfa_b200.h"
#include "fa_fwd_sm90.cuh"
#include "fa_splitkv_combine.cuh"

#include <cuda_runtime.h>

extern "C" void tfa_internal_count_launch(void);

namespace {

template <int D, bool CAUSAL, bool IS_BF16, bool OUT_F32>
cudaError_t launch(const CUtensorMap& tq, const CUtensorMap& tk, const CUtensorMap& tv, const tfa::FwdParams& p,
                   int nblocks, bool persist, cudaStream_t stream) {
  using C = tfa::FwdCfg<D>;
  auto kern = persist ? tfa::fa_fwd_sm90_kernel<D, CAUSAL, IS_BF16, OUT_F32, true, tfa::kVarlenCache>
                      : tfa::fa_fwd_sm90_kernel<D, CAUSAL, IS_BF16, OUT_F32, false, tfa::kVarlenCache>;
  const cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM_BYTES);
  if (e != cudaSuccess) return e;
  kern<<<nblocks, C::THREADS, C::SMEM_BYTES, stream>>>(tq, tk, tv, p);
  return cudaSuccess;
}

template <int D>
cudaError_t dispatch(bool causal, bool bf16, bool f32, const CUtensorMap& tq, const CUtensorMap& tk,
                     const CUtensorMap& tv, const tfa::FwdParams& p, int nblocks, bool persist, cudaStream_t s) {
#define TFA_GO(C_, B_, F_) return launch<D, C_, B_, F_>(tq, tk, tv, p, nblocks, persist, s)
  if (causal) {
    if (bf16) { if (f32) TFA_GO(true, true, true); else TFA_GO(true, true, false); }
    else      { if (f32) TFA_GO(true, false, true); else TFA_GO(true, false, false); }
  } else {
    if (bf16) { if (f32) TFA_GO(false, true, true); else TFA_GO(false, true, false); }
    else      { if (f32) TFA_GO(false, false, true); else TFA_GO(false, false, false); }
  }
#undef TFA_GO
}

}  // namespace

// The kVarlenCache forward over `nblocks` CTAs (the persistent kernel when `persist`), p.total_items work items; the
// caller sizes the grid and counts the launch.  Returns 0 or a cudaError_t.
int tfa_internal_launch_varlen_kvcache_fwd(int D, bool causal, bool bf16, bool f32, const CUtensorMap& tq,
                                           const CUtensorMap& tk, const CUtensorMap& tv, const tfa::FwdParams& p,
                                           int nblocks, bool persist, cudaStream_t stream) {
  const cudaError_t e = D == 64 ? dispatch<64>(causal, bf16, f32, tq, tk, tv, p, nblocks, persist, stream)
                                : dispatch<128>(causal, bf16, f32, tq, tk, tv, p, nblocks, persist, stream);
  return static_cast<int>(e);
}

// One launch over vp.ap.chunks 16-byte chunks, 256 per block; counted like every other launch.  Returns 0, a
// cudaError_t, or TFA_EINVAL_SHAPE when the grid does not fit.
int tfa_internal_launch_varlen_append(const tfa::VarlenAppendParams& vp, int D, cudaStream_t stream) {
  const long long blocks = (vp.ap.chunks + 255) / 256;
  if (blocks > 0x7fffffffLL) return TFA_EINVAL_SHAPE;
  auto kern = D == 64 ? tfa::kvcache_varlen_append_kernel<64> : tfa::kvcache_varlen_append_kernel<128>;
  kern<<<static_cast<int>(blocks), 256, 0, stream>>>(vp);
  tfa_internal_count_launch();
  return static_cast<int>(cudaGetLastError());
}

extern "C" {

// development aid (not in the public header): the length rule of the variable-length cache call on the host.
// out2 = {L, K}: the clamped cached length and the keys attended, for n query rows (n appended keys when append).
int tfa_internal_varlen_cache_lens(int raw, int capacity, int n, int append, int* out2) {
  tfa::varlen_cache_lens(raw, capacity, append ? n : 0, out2[0], out2[1]);
  return 0;
}
// development aid (not in the public header): where the variable-length append writes token i of sequence b at head
// h (raw = cache_seqlens[b], n = its appended rows), or -1 when the token is dropped
long long tfa_internal_varlen_append_offset(int raw, const int* block_table, long long bt_stride, int b, int i, int h,
                                            int page, int capacity, int n, int num_blocks, long long cs_b,
                                            long long cs_s, long long cs_h) {
  return tfa::varlen_append_offset(raw, block_table, bt_stride, b, i, h, page, capacity, n, num_blocks, cs_b, cs_s,
                                   cs_h);
}

}  // extern "C"
