// tfa_api.cu -- host side of the C ABI declared in include/tfa_b200.h.
//
// Replaces the reference's host dispatch chain
//   flash_attention_v2_cutlass -> set_params_fprop -> run_flash_attn_cutlass ->
//   FP16_SWITCH -> FWD_HEADDIM_SWITCH -> BOOL_SWITCH -> run_flash_fwd
// (/root/reference/flash_attention_cutlass/csrc/flash_attention.cu:320-361,687-772,
//  csrc/static_switch.h:17-66) for the sm_90a kernel in fa_fwd_sm90.cuh.
// Differences on purpose (SURVEY.md A.2): arguments are validated and rejected loudly, the
// caller's stream is honoured, nothing synchronises the device, nothing calls exit().
#include "../../include/tfa_b200.h"
#include "fa_fwd_launch.cuh"
#include "fa_kvcache_append.cuh"
#include "fa_splitkv_combine.cuh"

#include <cuda_runtime.h>
#include <cudaTypedefs.h>
#include <atomic>
#include <mutex>
#include <vector>
#include <cfloat>
#include <cmath>
#include <cstdlib>
#include <cstring>

// tfa_append.cu: the append's launch, compiled apart from the forward kernels
int tfa_internal_launch_append(const tfa::AppendKernelParams& p, const tfa::KvQuant* qs, bool q8, int D, bool bf16,
                               bool rotary, bool interleaved, cudaStream_t stream);

namespace {

using tfa::DebugRecord;
using tfa::FwdCfg;
using tfa::FwdParams;

std::atomic<unsigned long long> g_launches{0};
std::atomic<int> g_last_variant{0};         // kernel the last forward launch used (0 classic, 4 persistent)

// ---- driver entry point for cuTensorMapEncodeTiled (no link-time libcuda dependency) ----
PFN_cuTensorMapEncodeTiled_v12000 get_encode_fn() {
  static PFN_cuTensorMapEncodeTiled_v12000 fn = []() -> PFN_cuTensorMapEncodeTiled_v12000 {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres);
    if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess) return nullptr;
    return reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(p);
  }();
  return fn;
}

// ---- host-mapped watchdog record ----
DebugRecord* g_dbg_host = nullptr;
DebugRecord* g_dbg_dev = nullptr;
std::once_flag g_dbg_once;
void init_dbg() {
  std::call_once(g_dbg_once, [] {
    void* h = nullptr;
    if (cudaHostAlloc(&h, sizeof(DebugRecord), cudaHostAllocMapped | cudaHostAllocPortable) == cudaSuccess) {
      std::memset(h, 0, sizeof(DebugRecord));
      void* d = nullptr;
      if (cudaHostGetDevicePointer(&d, h, 0) == cudaSuccess) {
        g_dbg_host = static_cast<DebugRecord*>(h);
        g_dbg_dev = static_cast<DebugRecord*>(d);
      }
    }
  });
}

// (B?,H?,S,D)-strided 16-bit tensor -> 4-D tiled map with dims (D, S, H, B); the kernel addresses it as
// (x = head-dim offset, y = sequence row, z = head, w = batch).  Box = 64 x 128 elements, SWIZZLE_128B.
// dtype TFA_FP8_E4M3: a 1-byte (e4m3) cache, box = D x 128 bytes, unswizzled (the converter reads it row by row).
// `operand8`: a 1-byte tensor the 8-bit wgmma reads in place (kDenseFp8's Q and K), box = D x 128 bytes with the swizzle
// that matches its D-byte rows, SWIZZLE_128B (D = 128) or SWIZZLE_64B (D = 64).
int make_tmap(CUtensorMap* m, const void* base, int dtype, int D, int S, int B, int H, long long sb,
              long long sh, long long ss, bool operand8 = false) {
  const bool fp8 = dtype == TFA_FP8_E4M3;
  const CUtensorMapSwizzle swz = !fp8 ? CU_TENSOR_MAP_SWIZZLE_128B
                                 : !operand8 ? CU_TENSOR_MAP_SWIZZLE_NONE
                                 : D == 128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B;
  const int box_rows = 128, box_cols = fp8 ? D : 64;
  const cuuint64_t esz = fp8 ? 1 : 2;
  auto encode = get_encode_fn();
  if (!encode) return TFA_EDRIVER;
  const CUtensorMapDataType dt = fp8 ? CU_TENSOR_MAP_DATA_TYPE_UINT8
                                     : (dtype == TFA_BF16) ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16
                                                           : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
  const cuuint32_t box[4] = {static_cast<cuuint32_t>(box_cols), static_cast<cuuint32_t>(box_rows), 1, 1};
  const cuuint32_t estr[4] = {1, 1, 1, 1};
  const cuuint64_t dims[4] = {static_cast<cuuint64_t>(D), static_cast<cuuint64_t>(S), static_cast<cuuint64_t>(H),
                              static_cast<cuuint64_t>(B)};
  // size-1 dims may carry any stride; give them a legal one
  const cuuint64_t s1 = static_cast<cuuint64_t>(ss) * esz;
  const cuuint64_t s2 = (H > 1 ? static_cast<cuuint64_t>(sh) : static_cast<cuuint64_t>(ss) * S) * esz;
  const cuuint64_t s3 = (B > 1 ? static_cast<cuuint64_t>(sb) : s2 / esz * H) * esz;
  const cuuint64_t strides[3] = {s1, s2, s3};
  for (int i = 0; i < 3; ++i)
    if ((strides[i] % 16) || strides[i] >= (1ull << 40)) return TFA_EINVAL_STRIDE;
  CUresult r = encode(m, dt, 4, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swz,
                      CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : TFA_EDRIVER;
}

// ---- per-device state.  Function attributes, SM counts and workspaces belong to ONE device (context):
//      a process that drives several GPUs (tensors on cuda:0, then cuda:1) must not reuse the first device's. ----
constexpr int kMaxDevices = 64;
int current_device() {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= kMaxDevices) return -1;
  return dev;
}

int num_sms() {
  static std::atomic<int> cache[kMaxDevices];
  const int dev = current_device();
  if (dev < 0) return 0;
  int v = cache[dev].load(std::memory_order_relaxed);
  if (v == 0) {
    if (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) return 0;
    cache[dev].store(v, std::memory_order_relaxed);
  }
  return v;
}

// Kernel selection.  TFA_KERNEL (read once) forces one kernel: "classic" = one CTA per work item; "persist" = one CTA
// per SM walking the work items, whose producer loads the next item's Q and K/V while the current one finishes (same
// kernel source, fa_fwd_sm90.cuh, PERSIST = true).  Unset = AUTO: see choose_kernel().
enum { KV_AUTO = -1, KV_CLASSIC = 0, KV_PERSIST = 4 };
int kernel_variant() {
  static int v = [] {
    const char* e = std::getenv("TFA_KERNEL");
    if (e == nullptr) return static_cast<int>(KV_AUTO);
    if (std::strcmp(e, "classic") == 0) return static_cast<int>(KV_CLASSIC);
    if (std::strcmp(e, "persist") == 0) return static_cast<int>(KV_PERSIST);
    return static_cast<int>(KV_AUTO);
  }();
  return v;
}
// AUTO, from an A/B of the two schedules on one H100 80GB HBM3 at 700 W (profiles/h100_kernel_choice.txt): the persistent
// schedule wins on every non-causal shape measured (1-7 %) and on short causal items (S <= 1024: 11-17 %); from S = 4096
// up, causal items are unequal enough that the hardware's dynamic CTA scheduling wins (4-14 %).  The fused exchange keeps
// the persistent schedule (its multi-GPU timing has not been measured on H100).
int choose_kernel(bool causal, long long npairs, int n_extra) {
  const int forced = kernel_variant();
  if (forced != KV_AUTO) return forced;
  if (n_extra > 0 || !causal) return KV_PERSIST;
  return npairs <= 8 ? KV_PERSIST : KV_CLASSIC;
}

// Every launch ends here: count it (tfa_launch_count) and report a launch error.
int count_launch() {
  g_launches.fetch_add(1, std::memory_order_relaxed);
  return static_cast<int>(cudaGetLastError());
}

// The combine and append kernels: 256 threads per block, each block taking `per_block` of the `n` rows or chunks.
template <typename P>
int launch_small(void (*kern)(P), long long n, int per_block, const P& prm, cudaStream_t stream) {
  const long long blocks = (n + per_block - 1) / per_block;
  if (blocks > 0x7fffffffLL) return TFA_EINVAL_SHAPE;
  kern<<<static_cast<int>(blocks), 256, 0, stream>>>(prm);
  return count_launch();
}

// CTAs of a forward launch over `nitems` work items: one per item, or for the persistent schedule one per SM (0 when
// the SM count is unknown).  Records the schedule for tfa_internal_last_variant.
long long fwd_grid(long long nitems, int variant) {
  g_last_variant.store(variant, std::memory_order_relaxed);
  if (variant != KV_PERSIST) return nitems;
  const int sms = num_sms();
  if (sms <= 0) return 0;
  return nitems > sms ? sms : nitems;                                   // one CTA per SM
}

// One forward kernel launch over `nitems` work items of problem mode MODE (tfa::kDense / kVarlen / kCache /
// kVarlenCache / kCacheFp8 / kVarlenCacheFp8 / kDenseFp8 / kVarlenFp8 / kCacheQkv8 / kVarlenCacheQkv8).
template <int MODE>
int launch_fwd(int D, bool causal, bool bf16, bool f32, const CUtensorMap& tq, const CUtensorMap& tk,
               const CUtensorMap& tv, FwdParams p, long long nitems, int variant, cudaStream_t stream) {
  if (nitems > 0x3fffffffLL) return TFA_EINVAL_SHAPE;
  p.total_items = static_cast<int>(nitems);
  const long long nblocks = fwd_grid(nitems, variant);
  if (nblocks <= 0) return TFA_EARCH;
  const cudaError_t e = tfa::launch_forward<MODE>(D, causal, bf16, f32, tq, tk, tv, p, static_cast<int>(nblocks),
                                                  variant == KV_PERSIST, stream);
  return e != cudaSuccess ? static_cast<int>(e) : count_launch();
}

bool arch_ok() {
  static std::atomic<int> cache[kMaxDevices];    // 0 = unknown, 1 = sm_90, 2 = something else
  const int dev = current_device();
  if (dev < 0) return false;
  int v = cache[dev].load(std::memory_order_relaxed);
  if (v == 0) {
    int major = 0, minor = 0;     // sm_90a code (wgmma, setmaxnreg) runs on compute capability 9.0 only
    if (cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev) != cudaSuccess) return false;
    if (cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev) != cudaSuccess) return false;
    v = (major == 9 && minor == 0) ? 1 : 2;
    cache[dev].store(v, std::memory_order_relaxed);
  }
  return v == 1;
}

// The problem as the launcher sees it (superset of tfa_fwd_args / tfa_attn_args).
struct Problem {
  const void *q, *k, *v;
  void* out;
  float* lse;
  int B, Hq, Hkv, Sq, Sk, D;
  long long qsb, qsh, qss, ksb, ksh, kss;   // element strides of q and of k/v
  tfa::OutLayout ol;                        // where results go
  int dtype, causal;
  float scale;
  int out_fp32;
  int num_splits;
  void* ws;
  size_t ws_bytes;
  cudaStream_t stream;
  bool packed;                              // q / out / lse are packed rows: one batch entry of Sq = total_q rows
};

// The kernels take exponents in log2 units, c = fp32(scale * log2 e): a scale >= 0 is accepted while c is finite,
// i.e. up to about FLT_MAX / log2 e = 2.3587e38 (beyond it c = +inf turns every result into NaN).
constexpr float kLog2e = 1.4426950408889634f;
bool scale_in_range(float s) { return s >= 0.0f && std::isfinite(s * kLog2e); }

int validate(const Problem& a) {
  if (!a.q || !a.k || !a.v || !a.out) return TFA_EINVAL_PTR;
  if ((reinterpret_cast<uintptr_t>(a.q) | reinterpret_cast<uintptr_t>(a.k) | reinterpret_cast<uintptr_t>(a.v) |
       reinterpret_cast<uintptr_t>(a.out)) & 15u)
    return TFA_EINVAL_PTR;
  if (a.D != 64 && a.D != 128) return TFA_EINVAL_DIM;
  if (a.B < 1 || a.Hq < 1 || a.Hkv < 1 || a.Sq < 1 || a.Sk < 1) return TFA_EINVAL_SHAPE;
  if (a.Hq % a.Hkv) return TFA_EINVAL_HEADS;
  if (a.dtype != TFA_BF16 && a.dtype != TFA_FP16) return TFA_EINVAL_DTYPE;
  // the running max is taken on unscaled scores (as in the reference, flash_attention.cu:228,295): scale must be >= 0
  if (!scale_in_range(a.scale)) return TFA_EINVAL_SCALE;
  if (a.qss < a.D || (a.qss % 8) || (a.qsh % 8) || (a.qsb % 8)) return TFA_EINVAL_STRIDE;
  if (a.kss < a.D || (a.kss % 8) || (a.ksh % 8) || (a.ksb % 8)) return TFA_EINVAL_STRIDE;
  if (a.num_splits < 0) return TFA_EINVAL_SHAPE;
  return 0;
}

// Query rows of a dense call that see at least one key: causal with Sq > Sk leaves the first Sq - Sk rows without
// one.  The split count and the schedule are chosen for these rows: the items of the others load nothing.
int keyed_rows(bool causal, int Sq, int Sk) { return (causal && Sk < Sq) ? Sk : Sq; }

// Split-KV decision for the dense problem of S query rows per (batch, head) (a.Sq, or a packed call's max_seqlen_q).
// `want` 0 = auto: split only when the plain grid would leave more than half of the SMs idle, into as many splits as
// still fit one wave of CTAs (one CTA more than the SMs would double the time), each with >= 4 KV tiles;
// n > 1 = as asked, clamped so that no split is empty.
int resolve_splits(const Problem& a, int S, int want, int sms) {
  const long long items = ((static_cast<long long>(keyed_rows(a.causal != 0, S, a.Sk)) + 127) / 128) * a.B * a.Hq;
  const int nkv = (a.Sk + 127) / 128;
  int n = want;
  if (n == 0) {
    if (sms <= 0 || items * 2 > sms) return 1;
    n = static_cast<int>(sms / items);                  // floor: items * n CTAs must fit ONE wave
    if (n > nkv / 4) n = nkv / 4;
    if (n > 32) n = 32;
  }
  if (n > nkv) n = nkv;
  if (n < 2) return 1;
  const int tiles = (nkv + n - 1) / n;
  return (nkv + tiles - 1) / tiles;                                     // drop empty tail splits
}

// Split-KV workspace: `nsplit` normalised fp32 partials of the (B, Hq, S, D) output, then their nsplit (B, Hq, S)
// LSEs (set_output partitions it); packed, (Hq, total_q, D) partials and (Hq, total_q) LSEs.  Every split writes the
// LSEs of all rows it computes.
size_t splitkv_ws_bytes(const Problem& a, int nsplit) {
  if (nsplit <= 1) return 0;
  return static_cast<size_t>(nsplit) * (a.packed ? 1 : a.B) * a.Hq * a.Sq * (static_cast<size_t>(a.D) + 1) *
         sizeof(float);
}

struct SplitPlan {
  int nsplit;        // work items per Q-tile pair; > 1: partials in the workspace, merged by the combine
  int split_tiles;   // KV tiles per split
};

// The split count of a cache or dense call over S query rows per (batch, head).  Under auto (num_splits == 0) a
// missing, small or misaligned workspace means one pass; an asked-for count without its workspace is an error.
int plan_splits(const Problem& a, int S, SplitPlan& plan) {
  int nsplit = resolve_splits(a, S, a.num_splits, num_sms());
  if (nsplit > 1) {
    const size_t need = splitkv_ws_bytes(a, nsplit);
    const bool ws_ok = a.ws != nullptr && !(reinterpret_cast<uintptr_t>(a.ws) & 15u) && a.ws_bytes >= need;
    if (!ws_ok) {
      if (a.num_splits != 0) return TFA_EINVAL_WORKSPACE;
      nsplit = 1;                                      // auto: no workspace, no split
    }
  }
  const int nkv_total = (a.Sk + 127) / 128;
  plan.nsplit = nsplit;
  plan.split_tiles = (nkv_total + nsplit - 1) / nsplit;
  return 0;
}

// Where the forward over S query rows per (batch, head) writes: the caller's out / lse in one pass; with split-KV,
// contiguous (B, Hq, S, D) fp32 partials per split with their LSEs, which the combine merges into out / lse.  Packed:
// (Hq, total_q, D) partials, each sequence's rows at their packed offsets (the forward's ol.o(b, h, q0 + row)).
void set_output(FwdParams& p, const Problem& a, int S, int nsplit) {
  if (nsplit > 1) {
    const long long per_b = a.packed ? 0 : static_cast<long long>(a.Hq) * S;   // partial rows between batch entries
    const long long per_h = a.packed ? a.Sq : S;                                // between heads
    const long long rows = a.packed ? static_cast<long long>(a.Hq) * a.Sq : a.B * per_b;
    float* ws_o = static_cast<float*>(a.ws);
    p.out = nullptr;
    p.out_f32 = ws_o;
    p.lse = ws_o + static_cast<size_t>(nsplit) * rows * a.D;
    p.ol = {per_b * a.D, per_h * a.D, a.D, per_b, per_h};
    p.part_stride = rows * a.D;
    p.lse_part_stride = rows;
  } else {
    const bool f32 = a.out_fp32 != 0;
    p.out = f32 ? nullptr : a.out;
    p.out_f32 = f32 ? static_cast<float*>(a.out) : nullptr;
    p.lse = a.lse;
    p.ol = a.ol;
    p.part_stride = 0;
    p.lse_part_stride = 0;
  }
}

// the combine kernel takes D / 4 threads per row
template <int D, bool PACKED>
int launch_combine(const tfa::CombineParams& cp, bool bf16, bool f32, cudaStream_t stream) {
  auto kern = f32 ? tfa::splitkv_combine_kernel<D, true, true, PACKED>
                  : bf16 ? tfa::splitkv_combine_kernel<D, true, false, PACKED>
                         : tfa::splitkv_combine_kernel<D, false, false, PACKED>;
  return launch_small(kern, cp.rows, 256 / (D / 4), cp, stream);
}

// The rest of every forward call.  `p` arrives zeroed with its mode's fields set (Sk / causal_off / extra_dst, cu_q /
// cu_k, or the cache fields); this sets the fields all modes share, chooses the kernel, launches the forward over S
// query rows per (batch, head) and, with split-KV, the combine.
template <int MODE>
int run_forward(const Problem& a, FwdParams p, int S, const CUtensorMap& tq, const CUtensorMap& tk,
                const CUtensorMap& tv, SplitPlan plan) {
  const bool causal = a.causal != 0, bf16 = a.dtype == TFA_BF16, f32 = a.out_fp32 != 0;
  constexpr int M = tfa::base_mode(MODE);
  const long long npairs = (static_cast<long long>(S) + 127) / 128;
  // dense: the schedule is chosen for the Q-tile pairs with keys, as the split count is (resolve_splits)
  const int S_keyed = M == tfa::kDense ? keyed_rows(causal, S, a.Sk) : S;
  p.H = a.Hq;
  p.kv_group = a.Hq / a.Hkv;
  p.npairs = static_cast<int>(npairs);
  p.BH = a.B * a.Hq;
  p.head_chunk = p.BH < 8 ? p.BH : 8;
  p.scale = a.scale;
  // scale == 0 is legal (uniform attention over the visible keys): a tiny positive exponent scale keeps
  // masked scores at -inf (0 * -inf would be NaN) while every visible score still maps to exp2(0) = 1
  p.scale_log2 = fmaxf(a.scale * kLog2e, 1.0e-30f);
  p.m_none = -FLT_MAX / fmaxf(p.scale_log2, 1.0f);
  if (static_cast<double>(p.m_none) * fmaxf(p.scale_log2, 1.0f) < -static_cast<double>(FLT_MAX))
    p.m_none = std::nextafter(p.m_none, 0.0f);          // rounded toward zero: -m_none * c stays finite
  p.dbg = g_dbg_dev;
  p.S = S;
  p.nsplit = plan.nsplit;
  p.split_tiles = plan.split_tiles;
  set_output(p, a, S, plan.nsplit);

  const int variant = choose_kernel(causal, (static_cast<long long>(S_keyed) + 127) / 128, p.n_extra_dst);
  int rc = launch_fwd<MODE>(a.D, causal, bf16, f32 || plan.nsplit > 1, tq, tk, tv, p, npairs * a.B * a.Hq * plan.nsplit,
                            variant, a.stream);
  if (rc || plan.nsplit == 1) return rc;

  tfa::CombineParams cp;
  cp.o_part = p.out_f32;
  cp.lse_part = p.lse;
  cp.out = a.out;
  cp.lse = a.lse;
  cp.ol = a.ol;
  cp.nsplit = plan.nsplit;
  cp.H = a.Hq;
  if (a.packed) {         // one row per packed row of every head; a row outside its sequence's first S is not stored
    cp.rows = static_cast<long long>(a.Hq) * a.Sq;
    cp.S = a.Sq;
    cp.cu_q = p.cu_q; cp.B = a.B; cp.max_seqlen_q = S;
    return (a.D == 64) ? launch_combine<64, true>(cp, bf16, f32, a.stream)
                       : launch_combine<128, true>(cp, bf16, f32, a.stream);
  }
  cp.rows = static_cast<long long>(a.B) * a.Hq * S;
  cp.S = S;
  cp.cu_q = nullptr; cp.B = a.B; cp.max_seqlen_q = S;
  return (a.D == 64) ? launch_combine<64, false>(cp, bf16, f32, a.stream)
                     : launch_combine<128, false>(cp, bf16, f32, a.stream);
}

// The effective softmax scale s' of an FP8 call, as the caller rounds it from softmax_scale and the quantization scales,
// must stay a normal fp32 number (or 0 with softmax_scale = 0): an overflow, or an underflow that would silently turn
// the call into uniform attention, is TFA_EINVAL_SCALE.
int validate_fp8_scale(float softmax_scale, float s) {
  if (!scale_in_range(s)) return TFA_EINVAL_SCALE;
  if (softmax_scale > 0.0f && !(s >= FLT_MIN)) return TFA_EINVAL_SCALE;
  return 0;
}

// The FP8-attention arguments of a call whose 16-bit checks passed: the element type, the scales and q / k / v strides
// that keep every 1-byte TMA row and box 16-byte aligned.  Sets a.scale to s' = fp32(fp32(softmax_scale * q_scale) *
// k_scale).
int validate_qkv_quant(const tfa_qkv_quant_args& q, Problem& a) {
  if (q.qkv_dtype != TFA_FP8_E4M3) return TFA_EINVAL_QKVQUANT;
  for (const float x : {q.q_scale, q.k_scale, q.v_scale})
    if (!(x > 0.0f) || !std::isfinite(x)) return TFA_EINVAL_QKVQUANT;
  if ((a.qsb % 16) || (a.qsh % 16) || (a.qss % 16) || (a.ksb % 16) || (a.ksh % 16) || (a.kss % 16))
    return TFA_EINVAL_QKVQUANT;
  const float qs = a.scale * q.q_scale;
  const float s = qs * q.k_scale;
  if (int rc = validate_fp8_scale(a.scale, s)) return rc;
  a.scale = s;
  return 0;
}

Problem from_fwd_args(const tfa_fwd_args& a) {
  Problem q;
  q.q = a.q; q.k = a.k; q.v = a.v; q.out = a.out; q.lse = a.lse;
  q.B = a.B; q.Hq = a.H; q.Hkv = a.H; q.Sq = a.S; q.Sk = a.S; q.D = a.D;
  q.qsb = q.ksb = a.stride_b; q.qsh = q.ksh = a.stride_h; q.qss = q.kss = a.stride_s;
  q.ol = {a.stride_b, a.stride_h, a.stride_s, static_cast<long long>(a.H) * a.S, a.S};   // lse is (B, H, S)
  q.dtype = a.dtype; q.causal = a.is_causal; q.scale = a.softmax_scale; q.out_fp32 = a.out_fp32;
  q.num_splits = 1; q.ws = nullptr; q.ws_bytes = 0;
  q.stream = static_cast<cudaStream_t>(a.stream);
  q.packed = false;
  return q;
}

Problem from_attn_args(const tfa_attn_args& a) {
  Problem q;
  q.q = a.q; q.k = a.k; q.v = a.v; q.out = a.out; q.lse = a.lse;
  q.B = a.B; q.Hq = a.Hq; q.Hkv = a.Hkv; q.Sq = a.Sq; q.Sk = a.Sk; q.D = a.D;
  q.qsb = a.q_stride_b; q.qsh = a.q_stride_h; q.qss = a.q_stride_s;
  q.ksb = a.kv_stride_b; q.ksh = a.kv_stride_h; q.kss = a.kv_stride_s;
  q.ol = {q.qsb, q.qsh, q.qss, static_cast<long long>(a.Hq) * a.Sq, a.Sq};   // out as q, lse (B, Hq, Sq)
  q.dtype = a.dtype; q.causal = a.is_causal; q.scale = a.softmax_scale; q.out_fp32 = a.out_fp32;
  q.num_splits = a.num_splits; q.ws = a.workspace; q.ws_bytes = a.workspace_bytes;
  q.stream = static_cast<cudaStream_t>(a.stream);
  q.packed = false;
  return q;
}

// The packed tensors as one batch entry of total_q query rows and total_k keys (what validate() checks of them).
Problem from_varlen_args(const tfa_attn_varlen_args& a) {
  Problem q;
  q.q = a.q; q.k = a.k; q.v = a.v; q.out = a.out; q.lse = a.lse;
  q.B = a.B; q.Hq = a.Hq; q.Hkv = a.Hkv; q.Sq = a.total_q; q.Sk = a.total_k; q.D = a.D;
  q.qsb = 0; q.qsh = a.q_stride_h; q.qss = a.q_stride_s;
  q.ksb = 0; q.ksh = a.kv_stride_h; q.kss = a.kv_stride_s;
  q.ol = {0, a.D, static_cast<long long>(a.Hq) * a.D, 0, a.total_q};   // out (total_q, Hq, D), lse (Hq, total_q)
  q.dtype = a.dtype; q.causal = a.is_causal; q.scale = a.softmax_scale; q.out_fp32 = a.out_fp32;
  q.num_splits = 1; q.ws = nullptr; q.ws_bytes = 0;
  q.stream = static_cast<cudaStream_t>(a.stream);
  q.packed = true;
  return q;
}

// The cache problem as the dense one of Sk = capacity keys (what validate() and the split-KV helpers see of it).
Problem from_kvcache_args(const tfa_attn_kvcache_args& a) {
  Problem q;
  q.q = a.q; q.k = a.k_cache; q.v = a.v_cache; q.out = a.out; q.lse = a.lse;
  q.B = a.B; q.Hq = a.Hq; q.Hkv = a.Hkv; q.Sq = a.Sq; q.D = a.D;
  const long long cap = static_cast<long long>(a.max_blocks_per_seq) * a.page_block_size;
  q.Sk = cap > 0x7fffffffLL ? 0 : static_cast<int>(cap);          // 0 fails validate() as TFA_EINVAL_SHAPE
  q.qsb = a.q_stride_b; q.qsh = a.q_stride_h; q.qss = a.q_stride_s;
  q.ksb = a.cache_stride_block; q.ksh = a.cache_stride_h; q.kss = a.cache_stride_s;
  q.ol = {q.qsb, q.qsh, q.qss, static_cast<long long>(a.Hq) * a.Sq, a.Sq};   // out as q, lse (B, Hq, Sq)
  q.dtype = a.dtype; q.causal = a.is_causal; q.scale = a.softmax_scale; q.out_fp32 = a.out_fp32;
  q.num_splits = a.num_splits; q.ws = a.workspace; q.ws_bytes = a.workspace_bytes;
  q.stream = static_cast<cudaStream_t>(a.stream);
  q.packed = false;
  return q;
}

// The variable-length cache problem as the varlen one of total_q query rows (what validate() checks of q and out)
// against the cache of Sk = capacity keys.
Problem from_varlen_kvcache_args(const tfa_attn_varlen_kvcache_args& a) {
  Problem q;
  q.q = a.q; q.k = a.k_cache; q.v = a.v_cache; q.out = a.out; q.lse = a.lse;
  q.B = a.B; q.Hq = a.Hq; q.Hkv = a.Hkv; q.Sq = a.total_q; q.D = a.D;
  const long long cap = static_cast<long long>(a.max_blocks_per_seq) * a.page_block_size;
  q.Sk = cap > 0x7fffffffLL ? 0 : static_cast<int>(cap);          // 0 fails validate() as TFA_EINVAL_SHAPE
  q.qsb = 0; q.qsh = a.q_stride_h; q.qss = a.q_stride_s;
  q.ksb = a.cache_stride_block; q.ksh = a.cache_stride_h; q.kss = a.cache_stride_s;
  q.ol = {0, a.D, static_cast<long long>(a.Hq) * a.D, 0, a.total_q};   // out (total_q, Hq, D), lse (Hq, total_q)
  q.dtype = a.dtype; q.causal = a.is_causal; q.scale = a.softmax_scale; q.out_fp32 = a.out_fp32;
  q.num_splits = 1; q.ws = nullptr; q.ws_bytes = 0;
  q.stream = static_cast<cudaStream_t>(a.stream);
  q.packed = true;
  return q;
}

// The cache arguments of both cache calls: the lengths, the block table or the contiguous cache, k_new with v_new and
// their strides.  Only the dense-query call has Snew and a batch stride of k_new.
struct CacheArgs {
  void *k_cache, *v_cache;
  const void *k_new, *v_new;
  const int32_t *cache_seqlens, *block_table;
  int num_blocks, page_block_size, max_blocks_per_seq;
  long long block_table_stride, new_stride_s, new_stride_h;
  int Snew;                      // the dense-query call's
  long long new_stride_b;        // the dense-query call's
};

template <typename Args>
CacheArgs from_cache_args(const Args& ka) {
  CacheArgs c{};
  c.k_cache = ka.k_cache; c.v_cache = ka.v_cache; c.k_new = ka.k_new; c.v_new = ka.v_new;
  c.cache_seqlens = ka.cache_seqlens; c.block_table = ka.block_table;
  c.num_blocks = ka.num_blocks; c.page_block_size = ka.page_block_size; c.max_blocks_per_seq = ka.max_blocks_per_seq;
  c.block_table_stride = ka.block_table_stride; c.new_stride_s = ka.new_stride_s; c.new_stride_h = ka.new_stride_h;
  return c;
}

// Where a call's keys come from: the Problem's k / v tensors, packed ones through cu_seqlens_k, or the cache.
enum class Keys { kTensors, kPacked, kCache };

// A forward call: its Problem and what it asks for beyond it.  A null pointer: the call has no such part.
struct Call {
  Problem a;
  Keys keys;
  const int32_t* cu_seqlens_q = nullptr;     // a.packed: the sequences' query rows, at most max_seqlen_q each
  int max_seqlen_q = 0;
  const int32_t* cu_seqlens_k = nullptr;     // Keys::kPacked
  CacheArgs cache{};                          // Keys::kCache
  // the append also rotates q and k_new, and the forward reads its queries from rotary->q_rot (from q8 with q8)
  const tfa_rotary_args* rotary = nullptr;
  // an FP8 cache, into which the append quantizes and which the forward widens in shared memory
  const tfa_kv_quant_args* kv_quant = nullptr;
  // e4m3 q and K / V (or an FP8 cache) on 8-bit wgmma; a.dtype is the output's and k_new's
  const tfa_qkv_quant_args* qkv_quant = nullptr;
  // with qkv_quant, a 16-bit q: the append writes e4m3(q / q_scale) (rot(q) with rotary, rotary->q_rot unused) into
  // this contiguous scratch, the forward's q, whose layout the quantization checks see
  void* q8 = nullptr;
  void* const* extra_dst = nullptr;          // the fused exchange: n_extra more destinations of the output
  int n_extra = 0;
};

Call dense_call(const Problem& a, const tfa_qkv_quant_args* qkv_quant, void* const* extra_dst = nullptr,
                int n_extra = 0) {
  Call c{a, Keys::kTensors};
  c.qkv_quant = qkv_quant;
  c.extra_dst = extra_dst;
  c.n_extra = n_extra;
  return c;
}

Call varlen_call(const tfa_attn_varlen_args& va, const tfa_qkv_quant_args* qkv_quant) {
  Call c{from_varlen_args(va), Keys::kPacked};
  c.cu_seqlens_q = va.cu_seqlens_q; c.max_seqlen_q = va.max_seqlen_q; c.cu_seqlens_k = va.cu_seqlens_k;
  c.qkv_quant = qkv_quant;
  return c;
}

Call kvcache_call(const tfa_attn_kvcache_args& ka, const tfa_rotary_args* rotary, const tfa_kv_quant_args* kv_quant,
                  const tfa_qkv_quant_args* qkv_quant = nullptr, void* q8 = nullptr) {
  Call c{from_kvcache_args(ka), Keys::kCache};
  c.cache = from_cache_args(ka);
  c.cache.Snew = ka.Snew; c.cache.new_stride_b = ka.new_stride_b;
  c.rotary = rotary; c.kv_quant = kv_quant; c.qkv_quant = qkv_quant; c.q8 = q8;
  return c;
}

// `split` nullptr: one pass.  Otherwise split-KV as the dense-query call plans it, for the dense problem of
// max_seqlen_q rows per sequence, into packed partials.
Call varlen_kvcache_call(const tfa_attn_varlen_kvcache_args& va, const tfa_rotary_args* rotary,
                         const tfa_kv_quant_args* kv_quant, const tfa_qkv_quant_args* qkv_quant = nullptr,
                         void* q8 = nullptr, const tfa_split_args* split = nullptr) {
  Call c{from_varlen_kvcache_args(va), Keys::kCache};
  if (split) {
    c.a.num_splits = split->num_splits; c.a.ws = split->workspace; c.a.ws_bytes = split->workspace_bytes;
  }
  c.cu_seqlens_q = va.cu_seqlens_q; c.max_seqlen_q = va.max_seqlen_q;
  c.cache = from_cache_args(va);
  c.rotary = rotary; c.kv_quant = kv_quant; c.qkv_quant = qkv_quant; c.q8 = q8;
  return c;
}

// cu_seqlens_q of a packed query batch, a non-null 4-byte aligned pointer, and max_seqlen_q in [1, total_q].
int validate_seqlens_q(const Call& c) {
  if (!c.cu_seqlens_q || (reinterpret_cast<uintptr_t>(c.cu_seqlens_q) & 3u)) return TFA_EINVAL_SEQLENS;
  if (c.max_seqlen_q < 1 || c.max_seqlen_q > c.a.Sq) return TFA_EINVAL_SEQLENS;
  return 0;
}

// The cache arguments; Snew and the batch stride of k_new only for the dense-query call.
int validate_cache(const Call& c) {
  const CacheArgs& ka = c.cache;
  if (!ka.cache_seqlens || (reinterpret_cast<uintptr_t>(ka.cache_seqlens) & 3u) ||
      (reinterpret_cast<uintptr_t>(ka.block_table) & 3u))
    return TFA_EINVAL_KVCACHE;
  if (ka.num_blocks < 1 || ka.max_blocks_per_seq < 1 || ka.page_block_size < 1) return TFA_EINVAL_KVCACHE;
  if (ka.block_table) {
    if (ka.page_block_size % 128 || ka.block_table_stride < ka.max_blocks_per_seq) return TFA_EINVAL_KVCACHE;
  } else if (ka.max_blocks_per_seq != 1 || ka.num_blocks < c.a.B) {
    return TFA_EINVAL_KVCACHE;           // contiguous: one page (block b) per sequence
  }
  if ((ka.k_new == nullptr) != (ka.v_new == nullptr)) return TFA_EINVAL_KVCACHE;
  if (ka.k_new) {
    if (!c.a.packed) {
      const long long cap = static_cast<long long>(ka.max_blocks_per_seq) * ka.page_block_size;
      if (ka.Snew < 1 || ka.Snew > cap) return TFA_EINVAL_KVCACHE;
    }
    if ((reinterpret_cast<uintptr_t>(ka.k_new) | reinterpret_cast<uintptr_t>(ka.v_new)) & 15u) return TFA_EINVAL_PTR;
    if ((ka.new_stride_s % 8) || (ka.new_stride_h % 8) || ka.new_stride_s < 0 || ka.new_stride_h < 0)
      return TFA_EINVAL_STRIDE;
    if (!c.a.packed && ((ka.new_stride_b % 8) || ka.new_stride_b < 0)) return TFA_EINVAL_STRIDE;
  }
  return 0;
}

// The rotary arguments of a cache call whose cache arguments passed (capacity = a.Sk).  With q8 the call writes its
// rotated queries there and rotary->q_rot is not read.
int validate_rotary(const Call& c) {
  const tfa_rotary_args& ra = *c.rotary;
  if (!ra.cos || !ra.sin || ((reinterpret_cast<uintptr_t>(ra.cos) | reinterpret_cast<uintptr_t>(ra.sin)) & 15u))
    return TFA_EINVAL_ROTARY;
  if (!c.q8 && (!ra.q_rot || (reinterpret_cast<uintptr_t>(ra.q_rot) & 15u))) return TFA_EINVAL_ROTARY;
  if (ra.rotary_dim < 16 || ra.rotary_dim > c.a.D || ra.rotary_dim % 16) return TFA_EINVAL_ROTARY;
  if (ra.seqlen_ro < c.a.Sk) return TFA_EINVAL_ROTARY;    // every key position is below the capacity
  if (!c.cache.k_new) return TFA_EINVAL_ROTARY;            // as flash-attn: rotary rotates the appended keys
  return 0;
}

// The FP8-cache arguments of a cache call whose other arguments passed: the element type, the scales, and cache
// strides that keep every 1-byte TMA row and box 16-byte aligned.  Sets a.scale to the effective softmax scale
// s' = fp32(softmax_scale * k_scale), and `qs` to the scales.
int validate_quant(const tfa_kv_quant_args& q, Problem& a, tfa::KvQuant& qs) {
  if (q.cache_dtype != TFA_FP8_E4M3) return TFA_EINVAL_KVQUANT;
  if (!(q.k_scale > 0.0f) || !std::isfinite(q.k_scale) || !(q.v_scale > 0.0f) || !std::isfinite(q.v_scale))
    return TFA_EINVAL_KVQUANT;
  if ((a.ksb % 16) || (a.ksh % 16) || (a.kss % 16)) return TFA_EINVAL_KVQUANT;
  const float s = a.scale * q.k_scale;
  if (int rc = validate_fp8_scale(a.scale, s)) return rc;
  a.scale = s;
  qs.k_scale = q.k_scale;
  qs.v_scale = q.v_scale;
  return 0;
}

// The query side of an append that writes the queries the forward reads: rot(q) (`ra`), or with `q8` the e4m3 codes of
// q or rot(q) into q8.  Sets a.q to that scratch with its contiguous strides: (B, S, Hq, D), or packed (total_q, Hq, D)
// (S = max_seqlen_q rows of every sequence then).  out and lse keep their layout (a.ol).
void set_query_append(tfa::AppendKernelParams& rp, Problem& a, const tfa_rotary_args* ra, void* q8, int S) {
  rp.q = a.q; rp.q_rot = q8 ? q8 : ra->q_rot;
  rp.q_sb = a.packed ? 0 : a.qsb; rp.q_ss = a.qss; rp.q_sh = a.qsh;
  if (ra) {
    rp.cos = ra->cos; rp.sin = ra->sin;
    rp.rotary_dim = ra->rotary_dim; rp.seqlen_ro = ra->seqlen_ro;
  }
  rp.Sq = S; rp.Hq = a.Hq;
  rp.causal = a.causal != 0 ? 1 : 0;
  rp.q_chunks = static_cast<long long>(a.B) * S * a.Hq * (a.D / 8);
  a.q = rp.q_rot;
  a.qss = static_cast<long long>(a.Hq) * a.D;
  a.qsh = a.D;
  a.qsb = a.packed ? 0 : a.qss * a.Sq;
}

// The cache side of a cache call whose arguments passed (a = its Problem, capacity = a.Sk; `page` rows per K/V map
// entry): the key side of the append (ap.chunks = 0 without k_new) and the cache fields of the forward.  The
// dense-query call appends Snew rows of every sequence from (B, Snew, Hkv, D) k_new, and p.snew counts them; the
// variable-length call appends each sequence's n_b <= S rows, packed as q, and p.snew is a flag: sequence b appends as
// many keys as it has query rows.
void setup_cache(const Call& c, const Problem& a, int S, int page, tfa::AppendParams& ap, FwdParams& p) {
  const CacheArgs& ka = c.cache;
  const int n = a.packed ? S : ka.k_new ? ka.Snew : 0;
  ap.k_new = ka.k_new; ap.v_new = ka.v_new; ap.k_cache = ka.k_cache; ap.v_cache = ka.v_cache;
  ap.n_ss = ka.new_stride_s; ap.n_sh = ka.new_stride_h;
  if (a.packed) {
    ap.cu_q = c.cu_seqlens_q;
    ap.total_q = a.Sq;
  } else {
    ap.n_sb = ka.new_stride_b;
  }
  ap.c_sb = a.ksb; ap.c_ss = a.kss; ap.c_sh = a.ksh;
  ap.cache_seqlens = ka.cache_seqlens; ap.block_table = ka.block_table; ap.bt_stride = ka.block_table_stride;
  ap.page = page; ap.capacity = a.Sk; ap.snew = n; ap.num_blocks = ka.num_blocks; ap.Hkv = a.Hkv;
  ap.chunks = ka.k_new ? static_cast<long long>(a.B) * n * a.Hkv * (a.D / 8) : 0;
  p.cache_seqlens = ka.cache_seqlens;
  p.block_table = ka.block_table;
  p.bt_stride = ka.block_table_stride;
  p.page = page;
  p.capacity = a.Sk;
  p.snew = a.packed ? (ka.k_new ? 1 : 0) : n;
}

// How a call computes: on 16-bit operands, against an FP8 cache widened to 16 bits in shared memory, or with e4m3 q
// on 8-bit wgmma.
enum class Datapath { k16Bit, kFp8Cache, kE4m3 };

// The forward mode that solves `problem` (tfa::kDense / kVarlen / kCache / kVarlenCache) on `path`; -1: none does.
int forward_mode(int problem, Datapath path) {
  static constexpr int fp8_cache[4] = {-1, -1, tfa::kCacheFp8, tfa::kVarlenCacheFp8};
  static constexpr int e4m3[4] = {tfa::kDenseFp8, tfa::kVarlenFp8, tfa::kCacheQkv8, tfa::kVarlenCacheQkv8};
  return path == Datapath::k16Bit ? problem : path == Datapath::kFp8Cache ? fp8_cache[problem] : e4m3[problem];
}

// Every forward call.  Its checks run in this order, each only when the call has that part; they and the split plan
// come before anything is written, so a rejected call leaves the cache untouched.  Then the tensor maps, the append,
// the forward and, with split-KV, the combine.
int run_call(Call c) {
  Problem& a = c.a;
  const bool cache = c.keys == Keys::kCache;
  int rc;
  // the cache first: a table of 0 pages is a cache error, not a 0-key shape error
  if (cache && (rc = validate_cache(c))) return rc;
  if ((rc = validate(a))) return rc;
  if (a.packed && (rc = validate_seqlens_q(c))) return rc;
  if (c.keys == Keys::kPacked && (!c.cu_seqlens_k || (reinterpret_cast<uintptr_t>(c.cu_seqlens_k) & 3u)))
    return TFA_EINVAL_SEQLENS;
  if (c.rotary && (rc = validate_rotary(c))) return rc;
  // the query rows per (batch, head) the grid covers: packed, max_seqlen_q of every sequence (items past a sequence's
  // end return at once), and so do the append's query and key chunks (they return past n_b)
  const int S = a.packed ? c.max_seqlen_q : a.Sq;
  tfa::AppendKernelParams rp{};
  if (c.rotary || c.q8) set_query_append(rp, a, c.rotary, c.q8, S);
  tfa::KvQuant qs{1.0f, 1.0f};
  if (c.kv_quant && (rc = validate_quant(*c.kv_quant, a, qs))) return rc;
  if (c.qkv_quant) {
    if ((rc = validate_qkv_quant(*c.qkv_quant, a))) return rc;
    qs = tfa::KvQuant{c.qkv_quant->k_scale, c.qkv_quant->v_scale, c.qkv_quant->q_scale};
  }
  if (!arch_ok()) return TFA_EARCH;
  if (c.n_extra > 0) {
    // fused exchange: 16-bit output of the reference-shaped problem only, in one pass (tfa_fwd_args has no split
    // count: from_fwd_args asks for one)
    if (c.n_extra > 7 || c.extra_dst == nullptr || a.out_fp32 || a.Sq != a.Sk || a.Hq != a.Hkv || a.num_splits > 1)
      return TFA_EINVAL_SHAPE;
    for (int i = 0; i < c.n_extra; ++i)
      if (c.extra_dst[i] == nullptr || (reinterpret_cast<uintptr_t>(c.extra_dst[i]) & 15u)) return TFA_EINVAL_PTR;
  }
  init_dbg();

  // packed keys: one split holds every KV tile of any sequence.  Otherwise every split covers the same KV tiles of
  // every sequence, so a packed sequence with few keys fills only its first splits.
  SplitPlan plan{1, 0x7fffffff};
  if (c.keys != Keys::kPacked && (rc = plan_splits(a, S, plan))) return rc;

  // e4m3: the 8-bit swizzled Q and K maps the wgmma reads in place, the raw V map the converter transposes.  An FP8
  // cache: raw maps the converter widens.  A contiguous cache is one page of capacity rows per sequence.
  const Datapath path = c.qkv_quant ? Datapath::kE4m3 : c.kv_quant ? Datapath::kFp8Cache : Datapath::k16Bit;
  const bool e4m3 = path == Datapath::kE4m3;
  const int kv_dtype = path == Datapath::k16Bit ? a.dtype : TFA_FP8_E4M3;
  const int kv_rows = cache && c.cache.block_table ? c.cache.page_block_size : a.Sk;
  const int kv_b = cache ? c.cache.num_blocks : a.packed ? 1 : a.B;
  CUtensorMap tq, tk, tv;
  if ((rc = make_tmap(&tq, a.q, e4m3 ? TFA_FP8_E4M3 : a.dtype, a.D, a.Sq, a.packed ? 1 : a.B, a.Hq, a.qsb, a.qsh, a.qss,
                      e4m3)))
    return rc;
  if ((rc = make_tmap(&tk, a.k, kv_dtype, a.D, kv_rows, kv_b, a.Hkv, a.ksb, a.ksh, a.kss, e4m3))) return rc;
  if ((rc = make_tmap(&tv, a.v, kv_dtype, a.D, kv_rows, kv_b, a.Hkv, a.ksb, a.ksh, a.kss))) return rc;

  FwdParams p{};
  if (cache) {
    setup_cache(c, a, S, kv_rows, rp.ap, p);
    // rotary needs k_new (validate_rotary): every rotary call appends; a quantized q is written even without k_new
    if (c.cache.k_new || c.q8) {
      rc = tfa_internal_launch_append(rp, e4m3 || c.kv_quant ? &qs : nullptr, c.q8 != nullptr, a.D,
                                      a.dtype == TFA_BF16, c.rotary != nullptr, c.rotary && c.rotary->interleaved != 0,
                                      a.stream);
      if (rc) return rc;
    }
  }

  if (c.keys == Keys::kTensors) {
    p.Sk = a.Sk;
    p.causal_off = a.causal ? a.Sk - a.Sq : 0;            // < 0: the first Sq - Sk rows see no key
    p.keyless_pairs = p.causal_off < 0 ? -p.causal_off / 128 : 0;
    for (int i = 0; i < c.n_extra; ++i) p.extra_dst[i] = c.extra_dst[i];
    p.n_extra_dst = c.n_extra;
  }
  if (a.packed) {
    p.cu_q = c.cu_seqlens_q;
    p.total_q = a.Sq;
  }
  if (c.keys == Keys::kPacked) {
    p.cu_k = c.cu_seqlens_k;
    p.total_k = a.Sk;
  }
  if (path != Datapath::k16Bit) p.v_scale = qs.v_scale;

  const int problem = cache ? (a.packed ? tfa::kVarlenCache : tfa::kCache) : (a.packed ? tfa::kVarlen : tfa::kDense);
  switch (forward_mode(problem, path)) {
    case tfa::kDense: return run_forward<tfa::kDense>(a, p, S, tq, tk, tv, plan);
    case tfa::kVarlen: return run_forward<tfa::kVarlen>(a, p, S, tq, tk, tv, plan);
    case tfa::kCache: return run_forward<tfa::kCache>(a, p, S, tq, tk, tv, plan);
    case tfa::kVarlenCache: return run_forward<tfa::kVarlenCache>(a, p, S, tq, tk, tv, plan);
    case tfa::kCacheFp8: return run_forward<tfa::kCacheFp8>(a, p, S, tq, tk, tv, plan);
    case tfa::kVarlenCacheFp8: return run_forward<tfa::kVarlenCacheFp8>(a, p, S, tq, tk, tv, plan);
    case tfa::kDenseFp8: return run_forward<tfa::kDenseFp8>(a, p, S, tq, tk, tv, plan);
    case tfa::kVarlenFp8: return run_forward<tfa::kVarlenFp8>(a, p, S, tq, tk, tv, plan);
    case tfa::kCacheQkv8: return run_forward<tfa::kCacheQkv8>(a, p, S, tq, tk, tv, plan);
    case tfa::kVarlenCacheQkv8: return run_forward<tfa::kVarlenCacheQkv8>(a, p, S, tq, tk, tv, plan);
  }
  return TFA_EINVAL_KVQUANT;                            // an FP8 cache asked of keys that are not a cache
}

// ---- host-buffer path workspace ----
struct HostWs {
  void* d[4] = {nullptr, nullptr, nullptr, nullptr};   // q k v o
  float* dlse = nullptr;
  size_t bytes = 0, lse_bytes = 0;
  std::vector<cudaStream_t> streams;
  std::vector<cudaEvent_t> events;
};
HostWs g_ws_all[kMaxDevices];          // one per device: the buffers and streams belong to that device's context
std::mutex g_ws_mu;

void ws_release_locked(HostWs& g_ws) {
  for (auto& p : g_ws.d) { if (p) cudaFree(p); p = nullptr; }
  if (g_ws.dlse) cudaFree(g_ws.dlse);
  g_ws.dlse = nullptr;
  g_ws.bytes = g_ws.lse_bytes = 0;
  for (auto s : g_ws.streams) cudaStreamDestroy(s);
  g_ws.streams.clear();
}

}  // namespace

extern "C" {

int tfa_abi_version(void) { return TFA_ABI_VERSION; }

int tfa_fwd_ex(const tfa_fwd_args* args) {
  if (!args) return TFA_EINVAL_PTR;
  return run_call(dense_call(from_fwd_args(*args), nullptr));
}

int tfa_attn_fwd(const tfa_attn_args* args) {
  if (!args) return TFA_EINVAL_PTR;
  return run_call(dense_call(from_attn_args(*args), nullptr));
}

int tfa_attn_varlen_fwd(const tfa_attn_varlen_args* args) {
  if (!args) return TFA_EINVAL_PTR;
  return run_call(varlen_call(*args, nullptr));
}

int tfa_attn_kvcache_fwd(const tfa_attn_kvcache_args* args) {
  if (!args) return TFA_EINVAL_PTR;
  return run_call(kvcache_call(*args, nullptr, nullptr));
}

int tfa_attn_kvcache_rotary_fwd(const tfa_attn_kvcache_args* args, const tfa_rotary_args* rotary) {
  if (!args || !rotary) return TFA_EINVAL_PTR;
  return run_call(kvcache_call(*args, rotary, nullptr));
}

int tfa_attn_varlen_kvcache_fwd(const tfa_attn_varlen_kvcache_args* args) {
  if (!args) return TFA_EINVAL_PTR;
  return run_call(varlen_kvcache_call(*args, nullptr, nullptr));
}

int tfa_attn_varlen_kvcache_rotary_fwd(const tfa_attn_varlen_kvcache_args* args, const tfa_rotary_args* rotary,
                                       const tfa_kv_quant_args* quant) {
  if (!args || !rotary) return TFA_EINVAL_PTR;
  return run_call(varlen_kvcache_call(*args, rotary, quant));
}

int tfa_attn_kvcache_fp8_fwd(const tfa_attn_kvcache_args* args, const tfa_rotary_args* rotary,
                             const tfa_kv_quant_args* quant) {
  if (!args || !quant) return TFA_EINVAL_PTR;
  return run_call(kvcache_call(*args, rotary, quant));
}

int tfa_attn_varlen_kvcache_fp8_fwd(const tfa_attn_varlen_kvcache_args* args, const tfa_kv_quant_args* quant) {
  if (!args || !quant) return TFA_EINVAL_PTR;
  return run_call(varlen_kvcache_call(*args, nullptr, quant));
}

int tfa_attn_fp8_fwd(const tfa_attn_args* args, const tfa_qkv_quant_args* quant) {
  if (!args || !quant) return TFA_EINVAL_PTR;
  return run_call(dense_call(from_attn_args(*args), quant));
}

int tfa_attn_varlen_fp8_fwd(const tfa_attn_varlen_args* args, const tfa_qkv_quant_args* quant) {
  if (!args || !quant) return TFA_EINVAL_PTR;
  return run_call(varlen_call(*args, quant));
}

int tfa_attn_kvcache_qkv8_fwd(const tfa_attn_kvcache_args* args, const tfa_qkv_quant_args* quant) {
  if (!args || !quant) return TFA_EINVAL_PTR;
  return run_call(kvcache_call(*args, nullptr, nullptr, quant));
}

int tfa_attn_varlen_kvcache_qkv8_fwd(const tfa_attn_varlen_kvcache_args* args, const tfa_qkv_quant_args* quant) {
  if (!args || !quant) return TFA_EINVAL_PTR;
  return run_call(varlen_kvcache_call(*args, nullptr, nullptr, quant));
}

int tfa_attn_kvcache_qkv8_q16_fwd(const tfa_attn_kvcache_args* args, const tfa_rotary_args* rotary,
                                  const tfa_qkv_quant_args* quant, void* q8) {
  if (!args || !quant || !q8 || (reinterpret_cast<uintptr_t>(q8) & 15u)) return TFA_EINVAL_PTR;
  return run_call(kvcache_call(*args, rotary, nullptr, quant, q8));
}

int tfa_attn_varlen_kvcache_qkv8_q16_fwd(const tfa_attn_varlen_kvcache_args* args, const tfa_rotary_args* rotary,
                                         const tfa_qkv_quant_args* quant, void* q8) {
  if (!args || !quant || !q8 || (reinterpret_cast<uintptr_t>(q8) & 15u)) return TFA_EINVAL_PTR;
  return run_call(varlen_kvcache_call(*args, rotary, nullptr, quant, q8));
}

int tfa_attn_num_splits(const tfa_attn_args* args) {
  if (!args) return 1;
  const Problem a = from_attn_args(*args);
  if (a.B < 1 || a.Hq < 1 || a.Sq < 1 || a.Sk < 1 || a.num_splits < 0) return 1;
  return resolve_splits(a, a.Sq, a.num_splits, num_sms());
}

size_t tfa_attn_workspace_bytes(const tfa_attn_args* args, int num_splits) {
  if (!args || args->B < 1 || args->Hq < 1 || args->Sq < 1) return 0;
  return splitkv_ws_bytes(from_attn_args(*args), num_splits);
}

int tfa_attn_varlen_kvcache_split_fwd(const tfa_attn_varlen_kvcache_args* args, const tfa_rotary_args* rotary,
                                      const tfa_kv_quant_args* quant, const tfa_split_args* split) {
  if (!args || !split) return TFA_EINVAL_PTR;
  return run_call(varlen_kvcache_call(*args, rotary, quant, nullptr, nullptr, split));
}

int tfa_attn_varlen_kvcache_qkv8_split_fwd(const tfa_attn_varlen_kvcache_args* args, const tfa_rotary_args* rotary,
                                           const tfa_qkv_quant_args* quant, void* q8, const tfa_split_args* split) {
  if (!args || !quant || !split || (reinterpret_cast<uintptr_t>(q8) & 15u)) return TFA_EINVAL_PTR;
  if (!q8 && rotary) return TFA_EINVAL_ROTARY;          // an e4m3 q arrives quantized: nothing to rotate
  return run_call(varlen_kvcache_call(*args, rotary, nullptr, quant, q8, split));
}

// The dense problem (B, Hq, Sq = max_seqlen_q, Sk = capacity) of a variable-length cache call, for its split count.
int tfa_attn_varlen_kvcache_num_splits(const tfa_attn_varlen_kvcache_args* args, int num_splits) {
  if (!args) return 1;
  const Problem a = from_varlen_kvcache_args(*args);
  if (a.B < 1 || a.Hq < 1 || args->max_seqlen_q < 1 || a.Sk < 1 || num_splits < 0) return 1;
  return resolve_splits(a, args->max_seqlen_q, num_splits, num_sms());
}

size_t tfa_attn_varlen_kvcache_workspace_bytes(const tfa_attn_varlen_kvcache_args* args, int num_splits) {
  if (!args || args->Hq < 1 || args->total_q < 1 || args->D < 1) return 0;
  return splitkv_ws_bytes(from_varlen_kvcache_args(*args), num_splits);
}

int tfa_fwd_multi(const tfa_fwd_args* args, void* const* extra_out, int n_extra) {
  if (!args) return TFA_EINVAL_PTR;
  if (n_extra < 0) return TFA_EINVAL_SHAPE;
  return run_call(dense_call(from_fwd_args(*args), nullptr, extra_out, n_extra));
}

int tfa_fwd(const void* q, const void* k, const void* v, void* out, float* lse, int B, int H, int S, int D, int dtype,
            int is_causal, float softmax_scale, void* cuda_stream) {
  tfa_fwd_args a;
  std::memset(&a, 0, sizeof(a));
  a.q = q; a.k = k; a.v = v; a.out = out; a.lse = lse;
  a.B = B; a.H = H; a.S = S; a.D = D;
  a.stride_s = D;
  a.stride_h = static_cast<long long>(S) * D;
  a.stride_b = static_cast<long long>(H) * S * D;
  a.dtype = dtype;
  a.is_causal = is_causal;
  a.softmax_scale = softmax_scale;
  a.out_fp32 = 0;
  a.stream = cuda_stream;
  return run_call(dense_call(from_fwd_args(a), nullptr));
}

int tfa_fwd_host(const void* q, const void* k, const void* v, void* out, float* lse, int B, int H, int S, int D,
                 int dtype, int is_causal, float softmax_scale, int n_chunks) {
  if (!q || !k || !v || !out) return TFA_EINVAL_PTR;
  if (D != 64 && D != 128) return TFA_EINVAL_DIM;
  if (B < 1 || H < 1 || S < 1) return TFA_EINVAL_SHAPE;
  if (dtype != TFA_BF16 && dtype != TFA_FP16) return TFA_EINVAL_DTYPE;
  if (!scale_in_range(softmax_scale)) return TFA_EINVAL_SCALE;
  const int dev = current_device();
  if (dev < 0) return static_cast<int>(cudaErrorInvalidDevice);
  std::lock_guard<std::mutex> lk(g_ws_mu);
  HostWs& g_ws = g_ws_all[dev];
  const long long BH = static_cast<long long>(B) * H;
  const size_t head_bytes = static_cast<size_t>(S) * D * 2;
  const size_t total = head_bytes * BH;
  const size_t lse_total = static_cast<size_t>(BH) * S * sizeof(float);
  cudaError_t e;
  if (g_ws.bytes < total) {
    for (auto& p : g_ws.d) { if (p) cudaFree(p); p = nullptr; }
    g_ws.bytes = 0;
    for (auto& p : g_ws.d)
      if ((e = cudaMalloc(&p, total)) != cudaSuccess) { ws_release_locked(g_ws); return static_cast<int>(e); }
    g_ws.bytes = total;
  }
  if (g_ws.lse_bytes < lse_total) {
    if (g_ws.dlse) cudaFree(g_ws.dlse);
    g_ws.dlse = nullptr; g_ws.lse_bytes = 0;
    if ((e = cudaMalloc(reinterpret_cast<void**>(&g_ws.dlse), lse_total)) != cudaSuccess) return static_cast<int>(e);
    g_ws.lse_bytes = lse_total;
  }
  if (n_chunks < 1) n_chunks = 1;
  if (n_chunks > BH) n_chunks = static_cast<int>(BH);
  const int nstreams = n_chunks < 4 ? n_chunks : 4;
  while (static_cast<int>(g_ws.streams.size()) < nstreams) {
    cudaStream_t s;
    if ((e = cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking)) != cudaSuccess) return static_cast<int>(e);
    g_ws.streams.push_back(s);
  }
  // chunk over flattened (batch*head): every head is an independent problem
  int rc = 0;
  for (int c = 0; c < n_chunks && rc == 0; ++c) {
    const long long h0 = BH * c / n_chunks, h1 = BH * (c + 1) / n_chunks;
    const long long nh = h1 - h0;
    if (nh <= 0) continue;
    cudaStream_t s = g_ws.streams[c % nstreams];
    const size_t off = head_bytes * h0, nbytes = head_bytes * nh;
    const void* src[3] = {q, k, v};
    for (int i = 0; i < 3; ++i)
      if ((e = cudaMemcpyAsync(static_cast<char*>(g_ws.d[i]) + off, static_cast<const char*>(src[i]) + off, nbytes,
                               cudaMemcpyHostToDevice, s)) != cudaSuccess) { rc = static_cast<int>(e); break; }
    if (rc) break;
    rc = tfa_fwd(static_cast<char*>(g_ws.d[0]) + off, static_cast<char*>(g_ws.d[1]) + off,
                 static_cast<char*>(g_ws.d[2]) + off, static_cast<char*>(g_ws.d[3]) + off,
                 lse ? g_ws.dlse + h0 * S : nullptr, 1, static_cast<int>(nh), S, D, dtype, is_causal, softmax_scale, s);
    if (rc) break;
    if ((e = cudaMemcpyAsync(static_cast<char*>(out) + off, static_cast<char*>(g_ws.d[3]) + off, nbytes,
                             cudaMemcpyDeviceToHost, s)) != cudaSuccess) { rc = static_cast<int>(e); break; }
    if (lse && (e = cudaMemcpyAsync(lse + h0 * S, g_ws.dlse + h0 * S, static_cast<size_t>(nh) * S * sizeof(float),
                                    cudaMemcpyDeviceToHost, s)) != cudaSuccess) { rc = static_cast<int>(e); break; }
  }
  for (int i = 0; i < nstreams; ++i) {
    e = cudaStreamSynchronize(g_ws.streams[i]);
    if (e != cudaSuccess && rc == 0) rc = static_cast<int>(e);
  }
  if (rc != 0 && g_dbg_host && g_dbg_host->flag) rc = TFA_EDEVICE_FAULT;
  return rc;
}

void tfa_host_release(void) {
  const int dev = current_device();
  if (dev < 0) return;
  std::lock_guard<std::mutex> lk(g_ws_mu);
  ws_release_locked(g_ws_all[dev]);
}

unsigned long long tfa_launch_count(void) { return g_launches.load(); }
// development aid (not in the public header): which kernel the last forward launch used (0 classic, 4 persistent)
int tfa_internal_last_variant(void) { return g_last_variant.load(); }
// development aid (not in the public header): the kernel-selection rule of a dense call as a host function (no device
// needed); it takes the whole problem shape, of which the rule reads the mask, the rows with keys and the exchange
int tfa_internal_choose_kernel(int D, int causal, int Sq, int Sk, int B, int Hq, int nsplit, int sms, int n_extra) {
  (void)D; (void)B; (void)Hq; (void)nsplit; (void)sms;
  return choose_kernel(causal != 0, (static_cast<long long>(keyed_rows(causal != 0, Sq, Sk)) + 127) / 128, n_extra);
}
// exported for the self tests living in another translation unit
void tfa_internal_count_launch(void) { g_launches.fetch_add(1, std::memory_order_relaxed); }
void* tfa_internal_dbg_dev(void) { init_dbg(); return g_dbg_dev; }
void* tfa_internal_encode_fn(void) { return reinterpret_cast<void*>(get_encode_fn()); }

// development aid (not in the public header): the device's blockIdx -> work item mapping, callable on the host
int tfa_internal_decode_work(int block, int npairs, int nsplit, int head_chunk, int BH, int* out3) {
  int bh, split, pr;
  tfa::decode_work(block, npairs, nsplit, head_chunk, BH, bh, split, pr);
  out3[0] = bh; out3[1] = split; out3[2] = pr;
  return 0;
}

// development aid (not in the public header): the KV-cache address helpers of fa_fwd_sm90.cuh, callable on the host
// with host arrays.  out2 = {physical block, row} of key `key` of sequence b.
int tfa_internal_page_lookup(const int* block_table, long long bt_stride, int b, int key, int page, int* out2) {
  tfa::page_lookup(block_table, bt_stride, b, key, page, out2[0], out2[1]);
  return 0;
}
// The length rule and the append destination (cache_lens, append_offset), in the forms each cache call uses them; the
// exhaustive tests call both forms.  The dense-query call: the clamped cached length for snew <= capacity appended
// keys, and the destination of token i of sequence b read from cache_seqlens.
int tfa_internal_cache_len(int raw, int capacity, int snew) { return tfa::cache_len(raw, capacity, snew); }
long long tfa_internal_append_offset(const int* cache_seqlens, const int* block_table, long long bt_stride, int b,
                                     int i, int h, int page, int capacity, int snew, int num_blocks, long long cs_b,
                                     long long cs_s, long long cs_h) {
  return tfa::append_offset(cache_seqlens[b], block_table, bt_stride, b, i, h, page, capacity, snew, num_blocks, cs_b,
                            cs_s, cs_h);
}
// The variable-length call: out2 = {L, K} for n query rows (n appended keys when `append`, which may exceed the
// capacity), and the destination of token i (raw = cache_seqlens[b]), or -1 when the token is dropped.
int tfa_internal_varlen_cache_lens(int raw, int capacity, int n, int append, int* out2) {
  tfa::cache_lens(raw, capacity, append ? n : 0, out2[0], out2[1]);
  return 0;
}
long long tfa_internal_varlen_append_offset(int raw, const int* block_table, long long bt_stride, int b, int i, int h,
                                            int page, int capacity, int n, int num_blocks, long long cs_b,
                                            long long cs_s, long long cs_h) {
  return tfa::append_offset(raw, block_table, bt_stride, b, i, h, page, capacity, n, num_blocks, cs_b, cs_s, cs_h);
}
// development aid (not in the public header): the split-KV combine's packed row -> sequence rule on the host.
// out2 = {b, i}: packed row r is row i of sequence b; returns whether the combine merges it.
int tfa_internal_packed_row_seq(const int* cu, int B, int total, int S, int r, int* out2) {
  out2[0] = out2[1] = -1;
  return tfa::packed_row_seq(cu, B, total, S, r, out2[0], out2[1]) ? 1 : 0;
}
// development aid (not in the public header): the rotary position rule of fa_kvcache_append.cuh on the host
int tfa_internal_rotary_pos(int cache_len, int i, int causal, int is_query, int seqlen_ro) {
  return tfa::rotary_pos(cache_len, i, causal != 0, is_query != 0, seqlen_ro);
}
// development aid (not in the public header): the position rule of both cache calls (seq_rotary_pos) on the host --
// query row or appended key i of a sequence with raw = cache_seqlens[b] that appends n keys
int tfa_internal_seq_rotary_pos(int raw, int capacity, int n, int i, int causal, int is_query, int seqlen_ro) {
  return tfa::seq_rotary_pos(raw, capacity, n, i, causal != 0, is_query != 0, seqlen_ro);
}
// development aid (not in the public header): kDenseFp8's key order of P (fa_fwd_sm90.cuh) on the host -- pi of a
// 32-key block's A column, the accumulator element the packer puts into byte x of A register r, and the key the
// converter writes at position p of a V^T row
int tfa_internal_fp8_p_key(int c) { return tfa::fp8_p_key(c); }
int tfa_internal_fp8_pack_src(int r, int x) { return tfa::fp8_pack_src(r, x); }
int tfa_internal_fp8_vt_key(int p) { return tfa::fp8_vt_key(p); }

int tfa_debug_record(unsigned int out[8]) {
  if (!out) return TFA_EINVAL_PTR;
  if (!g_dbg_host) { std::memset(out, 0, 8 * sizeof(unsigned int)); return 0; }
  std::memcpy(out, g_dbg_host, 8 * sizeof(unsigned int));
  return 0;
}
void tfa_debug_clear(void) {
  if (g_dbg_host) std::memset(g_dbg_host, 0, sizeof(DebugRecord));
}

const char* tfa_error_string(int code) {
  switch (code) {
    case 0: return "success";
    case TFA_EINVAL_PTR: return "tfa: null or misaligned (16 B) pointer";
    case TFA_EINVAL_DIM: return "tfa: head_dim must be 64 or 128";
    case TFA_EINVAL_SHAPE: return "tfa: B, H, S must be >= 1 (and B*H*ceil(S/128) < 2^30); fused exchange needs the square MHA problem";
    case TFA_EINVAL_DTYPE: return "tfa: dtype must be TFA_BF16 (0) or TFA_FP16 (1)";
    case TFA_EINVAL_STRIDE: return "tfa: strides must be multiples of 8 elements with unit head_dim stride";
    case TFA_EDRIVER: return "tfa: cuTensorMapEncodeTiled unavailable or failed";
    case TFA_EARCH: return "tfa: this library only runs on compute capability 9.0 (H100, sm_90a)";
    case TFA_EDEVICE_FAULT: return "tfa: kernel watchdog fired (see tfa_debug_record)";
    case TFA_EINVAL_SCALE:
      return "tfa: softmax_scale (for FP8: the effective scale s') must be >= 0 with scale * log2(e) finite in fp32 "
             "(at most about 2.3587e38)";
    case TFA_EINVAL_HEADS: return "tfa: query heads must be a multiple of K/V heads";
    case TFA_EINVAL_WORKSPACE: return "tfa: split-KV needs a 16-byte aligned workspace of tfa_attn_workspace_bytes()";
    case TFA_EINVAL_SEQLENS:
      return "tfa: cu_seqlens must be non-null 4-byte aligned device pointers and max_seqlen_q in [1, total_q]";
    case TFA_EINVAL_KVCACHE:
      return "tfa: kv cache needs non-null 4-byte aligned cache_seqlens (block_table: aligned, page_block_size a "
             "multiple of 128), num_blocks and max_blocks_per_seq >= 1, and k_new with v_new, Snew in [1, capacity]";
    case TFA_EINVAL_ROTARY:
      return "tfa: rotary needs non-null 16-byte aligned cos, sin and q_rot, rotary_dim a multiple of 16 in [16, D], "
             "seqlen_ro >= capacity, and k_new";
    case TFA_EINVAL_KVQUANT:
      return "tfa: an FP8 cache needs cache_dtype TFA_FP8_E4M3 (2), finite k_scale and v_scale > 0, and cache strides "
             "that are multiples of 16 elements";
    case TFA_EINVAL_QKVQUANT:
      return "tfa: FP8 attention needs qkv_dtype TFA_FP8_E4M3 (2), finite q_scale, k_scale and v_scale > 0, and q / k / v "
             "strides that are multiples of 16 elements";
    default: return code > 0 ? cudaGetErrorString(static_cast<cudaError_t>(code)) : "tfa: unknown error";
  }
}

}  // extern "C"
