// attention_api.cpp -- the PyTorch-extension face of the library: Python module `attention_cutlass`.
//
// Mirrors the reference's operator surface so its own driver runs unchanged:
//   /root/reference/flash_attention_cutlass/csrc/attention_api.cpp:6-10   (PYBIND11_MODULE, one m.def)
//   /root/reference/flash_attention_cutlass/include/attention_api.h:10-11 (signature)
//   /root/reference/flash_attention_cutlass/csrc/flash_attention.cu:741-772 (host function)
//   /root/reference/flash_attention_cutlass/test.py:68,80                   (the only caller)
// i.e.  flash_attention_v2_cutlass(q, k, v, is_causal, softmax_scale) -> [out, softmax_lse]
// with q,k,v (B,H,S,D) contiguous CUDA fp16/bf16, out like q, softmax_lse (B,H,S) fp32.
//
// This file is host glue only: it validates, allocates the outputs with torch, and calls the
// C ABI (include/tfa_b200.h).  Deliberate differences from the reference (SURVEY.md A.2):
//   - launches on the CURRENT stream of q's device, under a device guard (ref: stream 0, no guard);
//   - no cudaDeviceSynchronize() (ref: flash_attention.cu:768);
//   - errors raise (TORCH_CHECK) instead of printf + exit(1) (ref: include/attention_api.cuh:20-29);
//   - dtype other than fp16/bf16 is rejected (ref silently treats everything non-bf16 as fp16, :351);
//   - bf16 is computed correctly (ref packs P to fp16 bits even in its bf16 branch, :206-215,:601).
#include <torch/extension.h>
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/tfa_b200.h"

namespace {

// same wording as the reference's CHECK_INPUT (include/attention_api.cuh:12-18)
#define TFA_CHECK_CUDA(x) TORCH_CHECK((x).device().is_cuda(), #x " must be a CUDA tensor")
#define TFA_CHECK_CONTIGUOUS(x) TORCH_CHECK((x).is_contiguous(), #x " must be contiguous")
#define TFA_CHECK_INPUT(x) \
  TFA_CHECK_CUDA(x);       \
  TFA_CHECK_CONTIGUOUS(x)

// NOTE: every message below is ONE preformatted string.  Multi-argument TORCH_CHECK formats through
// std::ostream inside this module, and this image's g++ emits weak libstdc++ stream symbols into the .so that
// crash once the CUDA user-mode driver is loaded (SIGSEGV in ostream::_M_insert<long>).
std::string fmt_msg(const char* fmt, long long a = 0, long long b = 0, long long c = 0, long long d = 0,
                    long long e = 0) {
  char buf[256];
  std::snprintf(buf, sizeof(buf), fmt, a, b, c, d, e);
  return std::string(buf);
}

// q is fp16 or bf16, and the other two tensors share its dtype and device; `names` names all three in the messages.
void check_dtype_device(const torch::Tensor& q, const torch::Tensor& k, const torch::Tensor& v,
                        const std::string& names) {
  TORCH_CHECK(q.scalar_type() == at::kHalf || q.scalar_type() == at::kBFloat16, "q must be float16 or bfloat16");
  TORCH_CHECK(k.scalar_type() == q.scalar_type() && v.scalar_type() == q.scalar_type(),
              names + " must have the same dtype");
  TORCH_CHECK(k.device() == q.device() && v.device() == q.device(), names + " must be on the same device");
}

void check_common(const torch::Tensor& q, const torch::Tensor& k, const torch::Tensor& v) {
  TORCH_CHECK(q.dim() == 4, fmt_msg("q must have 4 dimensions, got %lld", static_cast<long long>(q.dim())));
  check_dtype_device(q, k, v, "q, k, v");
  TORCH_CHECK(k.sizes() == q.sizes() && v.sizes() == q.sizes(),
              "q, k, v must have identical shapes (self-attention, Sq == Sk)");
}

// Split-KV of a dense problem: asks the library for the split count and, when it splits, allocates the workspace on
// q's device and sets num_splits / workspace / workspace_bytes in `a`.  Returns the workspace (undefined for one
// pass); the caller keeps it until the launch is enqueued.
torch::Tensor split_workspace(tfa_attn_args& a, const torch::Tensor& q) {
  torch::Tensor ws;
  const int nsplit = tfa_attn_num_splits(&a);
  if (nsplit > 1) {
    const size_t need = tfa_attn_workspace_bytes(&a, nsplit);
    ws = torch::empty({static_cast<int64_t>((need + 3) / 4)}, q.options().dtype(at::kFloat));
    a.workspace = ws.data_ptr();
    a.workspace_bytes = need;
    a.num_splits = nsplit;
  }
  return ws;
}

void raise_on_error(int rc) {
  if (rc == 0) return;
  if (rc == TFA_EDEVICE_FAULT) {
    unsigned int rec[8];
    tfa_debug_record(rec);
    TORCH_CHECK(false, std::string(tfa_error_string(rc)) +
                           fmt_msg(" [block %lld thread %lld site %lld iter %lld parity %lld]", rec[1], rec[2], rec[3],
                                   rec[4], rec[5]));
  }
  TORCH_CHECK(false, std::string("attention_cutlass: ") + tfa_error_string(rc) + fmt_msg(" (code %lld)", rc));
}

std::vector<torch::Tensor> fwd_generic(const torch::Tensor& q, const torch::Tensor& k, const torch::Tensor& v,
                                       bool is_causal, float softmax_scale, bool bshd, bool out_fp32) {
  check_common(q, k, v);
  const int64_t d0 = q.size(0), d1 = q.size(1), d2 = q.size(2), D = q.size(3);
  const int64_t B = d0, H = bshd ? d2 : d1, S = bshd ? d1 : d2;
  TORCH_CHECK(D == 64 || D == 128, fmt_msg("head_dim must be 64 or 128, got %lld", static_cast<long long>(D)));
  TORCH_CHECK(B >= 1 && H >= 1 && S >= 1, "empty tensors are not supported");

  torch::Tensor out, lse;
  int rc = 0;
  {
    // all validation happens above: nothing below throws while the device guard is live
    c10::cuda::CUDAGuard guard(q.device());
    out = out_fp32 ? torch::empty(q.sizes(), q.options().dtype(at::kFloat)) : torch::empty_like(q);
    lse = torch::empty({B, H, S}, q.options().dtype(at::kFloat));

    tfa_fwd_args a;
    a.q = q.data_ptr();
    a.k = k.data_ptr();
    a.v = v.data_ptr();
    a.out = out.data_ptr();
    a.lse = lse.data_ptr<float>();
    a.B = static_cast<int32_t>(B);
    a.H = static_cast<int32_t>(H);
    a.S = static_cast<int32_t>(S);
    a.D = static_cast<int32_t>(D);
    if (bshd) {
      a.stride_b = S * H * D; a.stride_s = H * D; a.stride_h = D;
    } else {
      a.stride_b = H * S * D; a.stride_h = S * D; a.stride_s = D;
    }
    a.dtype = q.scalar_type() == at::kBFloat16 ? TFA_BF16 : TFA_FP16;
    a.is_causal = is_causal ? 1 : 0;
    a.softmax_scale = softmax_scale;
    a.out_fp32 = out_fp32 ? 1 : 0;
    a.stream = at::cuda::getCurrentCUDAStream(q.device().index()).stream();
    rc = tfa_fwd_ex(&a);
  }
  raise_on_error(rc);
  return {out, lse};
}

}  // namespace

// The reference entry point (flash_attention.cu:741).  Positional-only, all five arguments
// required -- exactly what the reference's pybind registration yields (attention_api.cpp:8).
std::vector<torch::Tensor> flash_attention_v2_cutlass(torch::Tensor q, torch::Tensor k, torch::Tensor v,
                                                      bool is_causal, float softmax_scale) {
  TFA_CHECK_INPUT(q);
  TFA_CHECK_INPUT(k);
  TFA_CHECK_INPUT(v);
  return fwd_generic(q, k, v, is_causal, softmax_scale, /*bshd=*/false, /*out_fp32=*/false);
}

// (B,S,H,D) layout of the official flash_attn package (test.py:71-75 transposes into it);
// served by TMA strides, no transpose copy.
std::vector<torch::Tensor> flash_attention_v2_bshd(torch::Tensor q, torch::Tensor k, torch::Tensor v, bool is_causal,
                                                   float softmax_scale) {
  TFA_CHECK_INPUT(q);
  TFA_CHECK_INPUT(k);
  TFA_CHECK_INPUT(v);
  return fwd_generic(q, k, v, is_causal, softmax_scale, /*bshd=*/true, /*out_fp32=*/false);
}

// Validation build: identical kernel, epilogue skips the final 16-bit rounding (the idea of the
// reference's standalone DEBUG build, standalone_src/flash_attention_cutlass_standalone.cu:18-23,685-689).
std::vector<torch::Tensor> flash_attention_v2_fp32out(torch::Tensor q, torch::Tensor k, torch::Tensor v,
                                                      bool is_causal, float softmax_scale) {
  TFA_CHECK_INPUT(q);
  TFA_CHECK_INPUT(k);
  TFA_CHECK_INPUT(v);
  return fwd_generic(q, k, v, is_causal, softmax_scale, /*bshd=*/false, /*out_fp32=*/true);
}

// Generalised problem (SURVEY.md 8f rows 2-3): k, v are (B, Hkv, Sk, D) with Hq % Hkv == 0 and any Sk; causal is
// bottom-right aligned (flash_attention_c/csrc/attn.cpp:121-124; head grouping csrc/archive_)/attn.cpp:61,375).
// num_splits: 1 = single pass, n > 1 = split-KV with an LSE merge, 0 = let the library decide.
std::vector<torch::Tensor> flash_attention_v2_general(torch::Tensor q, torch::Tensor k, torch::Tensor v, bool is_causal,
                                                      float softmax_scale, int64_t num_splits) {
  TFA_CHECK_INPUT(q);
  TFA_CHECK_INPUT(k);
  TFA_CHECK_INPUT(v);
  TORCH_CHECK(q.dim() == 4 && k.dim() == 4 && v.dim() == 4, "q, k, v must have 4 dimensions");
  check_dtype_device(q, k, v, "q, k, v");
  TORCH_CHECK(k.sizes() == v.sizes(), "k and v must have identical shapes");
  TORCH_CHECK(k.size(0) == q.size(0) && k.size(3) == q.size(3), "k/v must share batch and head_dim with q");
  const int64_t B = q.size(0), Hq = q.size(1), Sq = q.size(2), D = q.size(3), Hkv = k.size(1), Sk = k.size(2);
  TORCH_CHECK(D == 64 || D == 128, fmt_msg("head_dim must be 64 or 128, got %lld", static_cast<long long>(D)));
  TORCH_CHECK(B >= 1 && Hq >= 1 && Hkv >= 1 && Sq >= 1 && Sk >= 1, "empty tensors are not supported");
  TORCH_CHECK(Hq % Hkv == 0, fmt_msg("query heads (%lld) must be a multiple of K/V heads (%lld)",
                                     static_cast<long long>(Hq), static_cast<long long>(Hkv)));
  TORCH_CHECK(num_splits >= 0 && num_splits <= 1024, "num_splits must be in [0, 1024]");

  torch::Tensor out, lse, ws;
  int rc = 0;
  {
    c10::cuda::CUDAGuard guard(q.device());
    out = torch::empty_like(q);
    lse = torch::empty({B, Hq, Sq}, q.options().dtype(at::kFloat));
    tfa_attn_args a;
    a.q = q.data_ptr(); a.k = k.data_ptr(); a.v = v.data_ptr();
    a.out = out.data_ptr(); a.lse = lse.data_ptr<float>();
    a.B = static_cast<int32_t>(B); a.Hq = static_cast<int32_t>(Hq); a.Hkv = static_cast<int32_t>(Hkv);
    a.Sq = static_cast<int32_t>(Sq); a.Sk = static_cast<int32_t>(Sk); a.D = static_cast<int32_t>(D);
    a.q_stride_b = Hq * Sq * D; a.q_stride_h = Sq * D; a.q_stride_s = D;
    a.kv_stride_b = Hkv * Sk * D; a.kv_stride_h = Sk * D; a.kv_stride_s = D;
    a.dtype = q.scalar_type() == at::kBFloat16 ? TFA_BF16 : TFA_FP16;
    a.is_causal = is_causal ? 1 : 0;
    a.softmax_scale = softmax_scale;
    a.out_fp32 = 0;
    a.num_splits = static_cast<int32_t>(num_splits);
    a.workspace = nullptr; a.workspace_bytes = 0;
    a.stream = at::cuda::getCurrentCUDAStream(q.device().index()).stream();
    ws = split_workspace(a, q);
    rc = tfa_attn_fwd(&a);
  }
  raise_on_error(rc);
  return {out, lse};
}

// FP8 attention (tfa_attn_fp8_fwd): q, k, v as flash_attention_v2_general but float8_e4m3fn, with the per-tensor scales
// their codes stand for; both products run on e4m3 tensor cores.  out_dtype (bfloat16 / float16) is the output's.
std::vector<torch::Tensor> flash_attention_v2_fp8(torch::Tensor q, torch::Tensor k, torch::Tensor v, double q_scale,
                                                  double k_scale, double v_scale, bool is_causal, float softmax_scale,
                                                  at::ScalarType out_dtype, int64_t num_splits) {
  TFA_CHECK_INPUT(q);
  TFA_CHECK_INPUT(k);
  TFA_CHECK_INPUT(v);
  TORCH_CHECK(q.dim() == 4 && k.dim() == 4 && v.dim() == 4, "q, k, v must have 4 dimensions");
  TORCH_CHECK(q.scalar_type() == at::kFloat8_e4m3fn && k.scalar_type() == at::kFloat8_e4m3fn &&
              v.scalar_type() == at::kFloat8_e4m3fn, "q, k, v must be float8_e4m3fn");
  TORCH_CHECK(k.device() == q.device() && v.device() == q.device(), "q, k, v must be on one device");
  TORCH_CHECK(out_dtype == at::kBFloat16 || out_dtype == at::kHalf, "out_dtype must be bfloat16 or float16");
  TORCH_CHECK(k.sizes() == v.sizes(), "k and v must have identical shapes");
  TORCH_CHECK(k.size(0) == q.size(0) && k.size(3) == q.size(3), "k/v must share batch and head_dim with q");
  const int64_t B = q.size(0), Hq = q.size(1), Sq = q.size(2), D = q.size(3), Hkv = k.size(1), Sk = k.size(2);
  TORCH_CHECK(D == 64 || D == 128, fmt_msg("head_dim must be 64 or 128, got %lld", static_cast<long long>(D)));
  TORCH_CHECK(B >= 1 && Hq >= 1 && Hkv >= 1 && Sq >= 1 && Sk >= 1, "empty tensors are not supported");
  TORCH_CHECK(Hq % Hkv == 0, fmt_msg("query heads (%lld) must be a multiple of K/V heads (%lld)",
                                     static_cast<long long>(Hq), static_cast<long long>(Hkv)));
  TORCH_CHECK(num_splits >= 0 && num_splits <= 1024, "num_splits must be in [0, 1024]");

  torch::Tensor out, lse, ws;
  int rc = 0;
  {
    c10::cuda::CUDAGuard guard(q.device());
    out = torch::empty(q.sizes(), q.options().dtype(out_dtype));
    lse = torch::empty({B, Hq, Sq}, q.options().dtype(at::kFloat));
    tfa_attn_args a;
    a.q = q.data_ptr(); a.k = k.data_ptr(); a.v = v.data_ptr();
    a.out = out.data_ptr(); a.lse = lse.data_ptr<float>();
    a.B = static_cast<int32_t>(B); a.Hq = static_cast<int32_t>(Hq); a.Hkv = static_cast<int32_t>(Hkv);
    a.Sq = static_cast<int32_t>(Sq); a.Sk = static_cast<int32_t>(Sk); a.D = static_cast<int32_t>(D);
    a.q_stride_b = Hq * Sq * D; a.q_stride_h = Sq * D; a.q_stride_s = D;
    a.kv_stride_b = Hkv * Sk * D; a.kv_stride_h = Sk * D; a.kv_stride_s = D;
    a.dtype = out_dtype == at::kBFloat16 ? TFA_BF16 : TFA_FP16;
    a.is_causal = is_causal ? 1 : 0;
    a.softmax_scale = softmax_scale;
    a.out_fp32 = 0;
    a.num_splits = static_cast<int32_t>(num_splits);
    a.workspace = nullptr; a.workspace_bytes = 0;
    a.stream = at::cuda::getCurrentCUDAStream(q.device().index()).stream();
    ws = split_workspace(a, q);
    tfa_qkv_quant_args qa{TFA_FP8_E4M3, static_cast<float>(q_scale), static_cast<float>(k_scale),
                          static_cast<float>(v_scale)};
    rc = tfa_attn_fp8_fwd(&a, &qa);
  }
  raise_on_error(rc);
  return {out, lse};
}

// Variable-length batch (the packed cu_seqlens interface of flash-attn's varlen forward): q (total_q, Hq, D),
// k, v (total_k, Hkv, D), unit head_dim stride (views of one packed (total, 3, H, D) qkv tensor need no copy);
// cu_seqlens_q / cu_seqlens_k int32 of B + 1 offsets on q's device.  Returns out (total_q, Hq, D) contiguous and
// lse (Hq, total_q).  max_seqlen_k is not taken: the kernel has no use for it.
std::vector<torch::Tensor> flash_attention_v2_varlen(torch::Tensor q, torch::Tensor k, torch::Tensor v,
                                                     torch::Tensor cu_seqlens_q, torch::Tensor cu_seqlens_k,
                                                     int64_t max_seqlen_q, bool is_causal, float softmax_scale) {
  TFA_CHECK_CUDA(q);
  TFA_CHECK_CUDA(k);
  TFA_CHECK_CUDA(v);
  TORCH_CHECK(q.dim() == 3 && k.dim() == 3 && v.dim() == 3, "q, k, v must have 3 dimensions (total, heads, head_dim)");
  check_dtype_device(q, k, v, "q, k, v");
  TORCH_CHECK(k.sizes() == v.sizes() && k.strides() == v.strides(), "k and v must have identical shapes and strides");
  TORCH_CHECK(k.size(2) == q.size(2), "k/v must share head_dim with q");
  TORCH_CHECK(q.stride(2) == 1 && k.stride(2) == 1, "q, k, v must have a unit head_dim stride");
  TORCH_CHECK(cu_seqlens_q.scalar_type() == at::kInt && cu_seqlens_k.scalar_type() == at::kInt,
              "cu_seqlens_q and cu_seqlens_k must be int32");
  TORCH_CHECK(cu_seqlens_q.device() == q.device() && cu_seqlens_k.device() == q.device(),
              "cu_seqlens_q and cu_seqlens_k must be on q's device");
  TORCH_CHECK(cu_seqlens_q.dim() == 1 && cu_seqlens_q.is_contiguous() && cu_seqlens_k.dim() == 1 &&
                  cu_seqlens_k.is_contiguous(),
              "cu_seqlens_q and cu_seqlens_k must be contiguous 1-D tensors");
  TORCH_CHECK(cu_seqlens_q.numel() >= 2 && cu_seqlens_k.numel() == cu_seqlens_q.numel(),
              fmt_msg("cu_seqlens_q and cu_seqlens_k must both hold B + 1 >= 2 offsets, got %lld and %lld",
                      static_cast<long long>(cu_seqlens_q.numel()), static_cast<long long>(cu_seqlens_k.numel())));
  const int64_t total_q = q.size(0), Hq = q.size(1), D = q.size(2), total_k = k.size(0), Hkv = k.size(1);
  const int64_t B = cu_seqlens_q.numel() - 1;
  TORCH_CHECK(D == 64 || D == 128, fmt_msg("head_dim must be 64 or 128, got %lld", static_cast<long long>(D)));
  TORCH_CHECK(total_q >= 1 && total_k >= 1 && Hq >= 1 && Hkv >= 1, "empty tensors are not supported");
  TORCH_CHECK(Hq % Hkv == 0, fmt_msg("query heads (%lld) must be a multiple of K/V heads (%lld)",
                                     static_cast<long long>(Hq), static_cast<long long>(Hkv)));
  TORCH_CHECK(max_seqlen_q >= 1 && max_seqlen_q <= total_q,
              fmt_msg("max_seqlen_q must be in [1, total_q = %lld], got %lld", static_cast<long long>(total_q),
                      static_cast<long long>(max_seqlen_q)));
  TORCH_CHECK(total_q < (1LL << 31) && total_k < (1LL << 31) && B < (1LL << 31), "tensors too large");

  torch::Tensor out, lse;
  int rc = 0;
  {
    c10::cuda::CUDAGuard guard(q.device());
    out = torch::empty({total_q, Hq, D}, q.options());
    lse = torch::empty({Hq, total_q}, q.options().dtype(at::kFloat));
    tfa_attn_varlen_args a;
    a.q = q.data_ptr(); a.k = k.data_ptr(); a.v = v.data_ptr();
    a.out = out.data_ptr(); a.lse = lse.data_ptr<float>();
    a.cu_seqlens_q = cu_seqlens_q.data_ptr<int32_t>();
    a.cu_seqlens_k = cu_seqlens_k.data_ptr<int32_t>();
    a.B = static_cast<int32_t>(B); a.Hq = static_cast<int32_t>(Hq); a.Hkv = static_cast<int32_t>(Hkv);
    a.D = static_cast<int32_t>(D);
    a.total_q = static_cast<int32_t>(total_q); a.total_k = static_cast<int32_t>(total_k);
    a.max_seqlen_q = static_cast<int32_t>(max_seqlen_q);
    a.q_stride_s = q.stride(0); a.q_stride_h = q.stride(1);
    a.kv_stride_s = k.stride(0); a.kv_stride_h = k.stride(1);
    a.dtype = q.scalar_type() == at::kBFloat16 ? TFA_BF16 : TFA_FP16;
    a.is_causal = is_causal ? 1 : 0;
    a.softmax_scale = softmax_scale;
    a.out_fp32 = 0;
    a.stream = at::cuda::getCurrentCUDAStream(q.device().index()).stream();
    rc = tfa_attn_varlen_fwd(&a);
  }
  raise_on_error(rc);
  return {out, lse};
}

// FP8 variable-length batch (tfa_attn_varlen_fp8_fwd): q, k, v as flash_attention_v2_varlen but float8_e4m3fn, with the
// per-tensor scales their codes stand for; both products run on e4m3 tensor cores.  out_dtype (bfloat16 / float16) is
// the output's.  Returns out (total_q, Hq, D) contiguous and lse (Hq, total_q).
std::vector<torch::Tensor> flash_attention_v2_varlen_fp8(torch::Tensor q, torch::Tensor k, torch::Tensor v,
                                                         torch::Tensor cu_seqlens_q, torch::Tensor cu_seqlens_k,
                                                         int64_t max_seqlen_q, double q_scale, double k_scale,
                                                         double v_scale, bool is_causal, float softmax_scale,
                                                         at::ScalarType out_dtype) {
  // the element types and devices first, then the CUDA checks: a wrong dtype is reported as such wherever q lives
  TORCH_CHECK(q.dim() == 3 && k.dim() == 3 && v.dim() == 3, "q, k, v must have 3 dimensions (total, heads, head_dim)");
  TORCH_CHECK(q.scalar_type() == at::kFloat8_e4m3fn && k.scalar_type() == at::kFloat8_e4m3fn &&
              v.scalar_type() == at::kFloat8_e4m3fn, "q, k, v must be float8_e4m3fn");
  TORCH_CHECK(out_dtype == at::kBFloat16 || out_dtype == at::kHalf, "out_dtype must be bfloat16 or float16");
  TORCH_CHECK(k.device() == q.device() && v.device() == q.device(), "q, k, v must be on the same device");
  TFA_CHECK_CUDA(q);
  TORCH_CHECK(k.sizes() == v.sizes() && k.strides() == v.strides(), "k and v must have identical shapes and strides");
  TORCH_CHECK(k.size(2) == q.size(2), "k/v must share head_dim with q");
  TORCH_CHECK(q.stride(2) == 1 && k.stride(2) == 1, "q, k, v must have a unit head_dim stride");
  TORCH_CHECK(cu_seqlens_q.scalar_type() == at::kInt && cu_seqlens_k.scalar_type() == at::kInt,
              "cu_seqlens_q and cu_seqlens_k must be int32");
  TORCH_CHECK(cu_seqlens_q.device() == q.device() && cu_seqlens_k.device() == q.device(),
              "cu_seqlens_q and cu_seqlens_k must be on q's device");
  TORCH_CHECK(cu_seqlens_q.dim() == 1 && cu_seqlens_q.is_contiguous() && cu_seqlens_k.dim() == 1 &&
                  cu_seqlens_k.is_contiguous(),
              "cu_seqlens_q and cu_seqlens_k must be contiguous 1-D tensors");
  TORCH_CHECK(cu_seqlens_q.numel() >= 2 && cu_seqlens_k.numel() == cu_seqlens_q.numel(),
              fmt_msg("cu_seqlens_q and cu_seqlens_k must both hold B + 1 >= 2 offsets, got %lld and %lld",
                      static_cast<long long>(cu_seqlens_q.numel()), static_cast<long long>(cu_seqlens_k.numel())));
  const int64_t total_q = q.size(0), Hq = q.size(1), D = q.size(2), total_k = k.size(0), Hkv = k.size(1);
  const int64_t B = cu_seqlens_q.numel() - 1;
  TORCH_CHECK(D == 64 || D == 128, fmt_msg("head_dim must be 64 or 128, got %lld", static_cast<long long>(D)));
  TORCH_CHECK(total_q >= 1 && total_k >= 1 && Hq >= 1 && Hkv >= 1, "empty tensors are not supported");
  TORCH_CHECK(Hq % Hkv == 0, fmt_msg("query heads (%lld) must be a multiple of K/V heads (%lld)",
                                     static_cast<long long>(Hq), static_cast<long long>(Hkv)));
  TORCH_CHECK(max_seqlen_q >= 1 && max_seqlen_q <= total_q,
              fmt_msg("max_seqlen_q must be in [1, total_q = %lld], got %lld", static_cast<long long>(total_q),
                      static_cast<long long>(max_seqlen_q)));
  TORCH_CHECK(total_q < (1LL << 31) && total_k < (1LL << 31) && B < (1LL << 31), "tensors too large");

  torch::Tensor out, lse;
  int rc = 0;
  {
    c10::cuda::CUDAGuard guard(q.device());
    out = torch::empty({total_q, Hq, D}, q.options().dtype(out_dtype));
    lse = torch::empty({Hq, total_q}, q.options().dtype(at::kFloat));
    tfa_attn_varlen_args a;
    a.q = q.data_ptr(); a.k = k.data_ptr(); a.v = v.data_ptr();
    a.out = out.data_ptr(); a.lse = lse.data_ptr<float>();
    a.cu_seqlens_q = cu_seqlens_q.data_ptr<int32_t>();
    a.cu_seqlens_k = cu_seqlens_k.data_ptr<int32_t>();
    a.B = static_cast<int32_t>(B); a.Hq = static_cast<int32_t>(Hq); a.Hkv = static_cast<int32_t>(Hkv);
    a.D = static_cast<int32_t>(D);
    a.total_q = static_cast<int32_t>(total_q); a.total_k = static_cast<int32_t>(total_k);
    a.max_seqlen_q = static_cast<int32_t>(max_seqlen_q);
    a.q_stride_s = q.stride(0); a.q_stride_h = q.stride(1);
    a.kv_stride_s = k.stride(0); a.kv_stride_h = k.stride(1);
    a.dtype = out_dtype == at::kBFloat16 ? TFA_BF16 : TFA_FP16;
    a.is_causal = is_causal ? 1 : 0;
    a.softmax_scale = softmax_scale;
    a.out_fp32 = 0;
    a.stream = at::cuda::getCurrentCUDAStream(q.device().index()).stream();
    tfa_qkv_quant_args qa{TFA_FP8_E4M3, static_cast<float>(q_scale), static_cast<float>(k_scale),
                          static_cast<float>(v_scale)};
    rc = tfa_attn_varlen_fp8_fwd(&a, &qa);
  }
  raise_on_error(rc);
  return {out, lse};
}

namespace {

// The cache's shape as the cache entry points pass it to the library.
struct CacheShape {
  int64_t nblk, page, Hkv, mbps, bts;
};

// The arguments both cache entry points share, for a q of B sequences: the caches, cache_seqlens, block_table and the
// pairing, device and dtype of k_new / v_new.  Each entry point checks the shapes of its q and k_new itself.  Throws
// on a bad argument, before any device work.  `fp8`: the caches are float8_e4m3fn (the FP8 entry points), else q's
// dtype.
CacheShape check_cache(const torch::Tensor& q, int64_t B, const torch::Tensor& k_cache, const torch::Tensor& v_cache,
                       const torch::Tensor& cache_seqlens, const std::optional<torch::Tensor>& block_table,
                       const std::optional<torch::Tensor>& k_new, const std::optional<torch::Tensor>& v_new,
                       bool fp8 = false) {
  TFA_CHECK_CUDA(k_cache);
  TFA_CHECK_CUDA(v_cache);
  TORCH_CHECK(k_cache.dim() == 4 && v_cache.dim() == 4, "k_cache, v_cache must have 4 dimensions");
  if (fp8) {
    TORCH_CHECK(q.scalar_type() == at::kHalf || q.scalar_type() == at::kBFloat16, "q must be float16 or bfloat16");
    TORCH_CHECK(k_cache.scalar_type() == at::kFloat8_e4m3fn && v_cache.scalar_type() == at::kFloat8_e4m3fn,
                "k_cache and v_cache must be float8_e4m3fn for the FP8 cache calls");
    TORCH_CHECK(k_cache.device() == q.device() && v_cache.device() == q.device(),
                "q, k_cache, v_cache must be on the same device");
  } else {
    check_dtype_device(q, k_cache, v_cache, "q, k_cache, v_cache");
  }
  TORCH_CHECK(k_cache.sizes() == v_cache.sizes() && k_cache.strides() == v_cache.strides(),
              "k_cache and v_cache must have identical shapes and strides");
  TORCH_CHECK(q.stride(-1) == 1 && k_cache.stride(3) == 1, "q and the caches must have a unit head_dim stride");
  TORCH_CHECK(k_cache.size(3) == q.size(-1), "the caches must share head_dim with q");
  TORCH_CHECK(cache_seqlens.scalar_type() == at::kInt && cache_seqlens.device() == q.device() &&
                  cache_seqlens.dim() == 1 && cache_seqlens.is_contiguous() && cache_seqlens.numel() == B,
              "cache_seqlens must be a contiguous int32 (B,) tensor on q's device");
  CacheShape c{k_cache.size(0), k_cache.size(1), k_cache.size(2), 1, 1};
  if (block_table.has_value()) {
    const torch::Tensor& bt = *block_table;
    TORCH_CHECK(bt.scalar_type() == at::kInt && bt.device() == q.device() && bt.dim() == 2 && bt.size(0) == B &&
                    bt.stride(1) == 1,
                "block_table must be an int32 (B, max_blocks_per_seq) tensor on q's device with unit column stride");
    TORCH_CHECK(c.page % 128 == 0, fmt_msg("a paged cache needs page_block_size % 128 == 0, got %lld",
                                           static_cast<long long>(c.page)));
    c.mbps = bt.size(1);
    c.bts = bt.stride(0);
  } else {
    TORCH_CHECK(c.nblk == B, "without block_table the caches must be (B, capacity, Hkv, D)");
  }
  TORCH_CHECK(k_new.has_value() == v_new.has_value(), "k_new and v_new must be given together");
  if (k_new.has_value()) {
    const torch::Tensor &kn = *k_new, &vn = *v_new;
    TORCH_CHECK(kn.device() == q.device() && vn.device() == q.device() && kn.scalar_type() == q.scalar_type() &&
                    vn.scalar_type() == q.scalar_type(),
                "k_new and v_new must be on q's device with q's dtype");
  }
  return c;
}

// A KV-cache call's tensors after check_kvcache(): the optional ones resolved, and the shape facts the fill needs.
struct KvcacheCall {
  torch::Tensor q, k_cache, v_cache, cache_seqlens;
  std::optional<torch::Tensor> block_table, k_new, v_new;
  int64_t B, Sq, Hq, D, nblk, page, Hkv, mbps, bts, snew;
};

// Every check of a KV-cache call; throws on a bad argument, before any device work.
KvcacheCall check_kvcache(const torch::Tensor& q, const torch::Tensor& k_cache, const torch::Tensor& v_cache,
                          const torch::Tensor& cache_seqlens, const std::optional<torch::Tensor>& block_table,
                          const std::optional<torch::Tensor>& k_new, const std::optional<torch::Tensor>& v_new,
                          int64_t num_splits, bool fp8 = false) {
  TFA_CHECK_CUDA(q);
  TORCH_CHECK(q.dim() == 4, "q must have 4 dimensions (B, Sq, Hq, D)");
  const CacheShape cs = check_cache(q, q.size(0), k_cache, v_cache, cache_seqlens, block_table, k_new, v_new, fp8);
  KvcacheCall c{q, k_cache, v_cache, cache_seqlens, block_table, k_new, v_new};
  c.B = q.size(0); c.Sq = q.size(1); c.Hq = q.size(2); c.D = q.size(3);
  c.nblk = cs.nblk; c.page = cs.page; c.Hkv = cs.Hkv; c.mbps = cs.mbps; c.bts = cs.bts;
  c.snew = 0;
  if (k_new.has_value()) {
    const torch::Tensor &kn = *k_new, &vn = *v_new;
    TORCH_CHECK(kn.dim() == 4 && kn.sizes() == vn.sizes() && kn.strides() == vn.strides() && kn.size(0) == c.B &&
                    kn.size(2) == c.Hkv && kn.size(3) == c.D && kn.stride(3) == 1,
                "k_new and v_new must be (B, Snew, Hkv, D) with identical strides and a unit head_dim stride");
    c.snew = kn.size(1);
    TORCH_CHECK(c.snew >= 1 && c.snew <= c.mbps * c.page, "Snew must be in [1, capacity]");
  }
  TORCH_CHECK(c.D == 64 || c.D == 128, fmt_msg("head_dim must be 64 or 128, got %lld", static_cast<long long>(c.D)));
  TORCH_CHECK(c.B >= 1 && c.Sq >= 1 && c.Hq >= 1 && c.Hkv >= 1, "empty tensors are not supported");
  TORCH_CHECK(c.Hq % c.Hkv == 0, fmt_msg("query heads (%lld) must be a multiple of K/V heads (%lld)",
                                         static_cast<long long>(c.Hq), static_cast<long long>(c.Hkv)));
  TORCH_CHECK(num_splits >= 0 && num_splits <= 1024, "num_splits must be in [0, 1024]");
  return c;
}

// The dense-query cache call once every argument passed: allocates out (q's strides; a non-dense q is replaced by its
// contiguous copy first), lse, the split-KV workspace and, with rotary (`r`), q_rot, and runs the call.  `quant`
// nullptr: a 16-bit cache.
std::vector<torch::Tensor> kvcache_fwd(KvcacheCall& c, bool is_causal, float softmax_scale, int64_t num_splits,
                                       tfa_rotary_args* r, const tfa_kv_quant_args* quant) {
  torch::Tensor out, lse, ws, q_rot;
  int rc = 0;
  {
    c10::cuda::CUDAGuard guard(c.q.device());
    out = torch::empty_like(c.q);
    if (out.strides() != c.q.strides()) {     // out takes q's strides: give a non-dense q out's dense ones
      c.q = c.q.contiguous();
      out = torch::empty_like(c.q);
    }
    lse = torch::empty({c.B, c.Hq, c.Sq}, c.q.options().dtype(at::kFloat));
    tfa_attn_kvcache_args a;
    std::memset(&a, 0, sizeof(a));
    a.q = c.q.data_ptr(); a.k_cache = c.k_cache.data_ptr(); a.v_cache = c.v_cache.data_ptr();
    a.k_new = c.snew ? c.k_new->data_ptr() : nullptr;
    a.v_new = c.snew ? c.v_new->data_ptr() : nullptr;
    a.out = out.data_ptr(); a.lse = lse.data_ptr<float>();
    a.cache_seqlens = c.cache_seqlens.data_ptr<int32_t>();
    a.block_table = c.block_table.has_value() ? c.block_table->data_ptr<int32_t>() : nullptr;
    a.B = static_cast<int32_t>(c.B); a.Hq = static_cast<int32_t>(c.Hq); a.Hkv = static_cast<int32_t>(c.Hkv);
    a.Sq = static_cast<int32_t>(c.Sq); a.D = static_cast<int32_t>(c.D);
    a.num_blocks = static_cast<int32_t>(c.nblk); a.page_block_size = static_cast<int32_t>(c.page);
    a.max_blocks_per_seq = static_cast<int32_t>(c.mbps); a.Snew = static_cast<int32_t>(c.snew);
    a.q_stride_b = c.q.stride(0); a.q_stride_s = c.q.stride(1); a.q_stride_h = c.q.stride(2);
    a.cache_stride_block = c.k_cache.stride(0); a.cache_stride_s = c.k_cache.stride(1);
    a.cache_stride_h = c.k_cache.stride(2);
    a.block_table_stride = c.bts;
    if (c.snew) {
      a.new_stride_b = c.k_new->stride(0); a.new_stride_s = c.k_new->stride(1); a.new_stride_h = c.k_new->stride(2);
    }
    a.dtype = c.q.scalar_type() == at::kBFloat16 ? TFA_BF16 : TFA_FP16;
    a.is_causal = is_causal ? 1 : 0;
    a.softmax_scale = softmax_scale;
    a.num_splits = static_cast<int32_t>(num_splits);
    a.stream = at::cuda::getCurrentCUDAStream(c.q.device().index()).stream();
    // split count and workspace: those of the dense problem with Sk = capacity
    tfa_attn_args d;
    std::memset(&d, 0, sizeof(d));
    d.B = a.B; d.Hq = a.Hq; d.Hkv = a.Hkv; d.Sq = a.Sq; d.D = a.D;
    d.Sk = static_cast<int32_t>(std::min<int64_t>(c.mbps * c.page, 0x7fffffff));
    d.is_causal = a.is_causal;
    d.num_splits = a.num_splits;
    ws = split_workspace(d, c.q);
    a.num_splits = d.num_splits; a.workspace = d.workspace; a.workspace_bytes = d.workspace_bytes;
    if (r) {
      q_rot = torch::empty({c.B, c.Sq, c.Hq, c.D}, c.q.options().memory_format(at::MemoryFormat::Contiguous));
      r->q_rot = q_rot.data_ptr();
    }
    rc = quant ? tfa_attn_kvcache_fp8_fwd(&a, r, quant)
         : r   ? tfa_attn_kvcache_rotary_fwd(&a, r)
               : tfa_attn_kvcache_fwd(&a);
  }
  raise_on_error(rc);
  return {out, lse};
}

}  // namespace

// Attention against a KV cache (flash-attn's flash_attn_with_kvcache without rotary): q (B, Sq, Hq, D);
// k_cache / v_cache (num_blocks, page_block_size, Hkv, D) with block_table int32 (B, max_blocks_per_seq), or a
// contiguous (B, capacity, Hkv, D) cache with block_table None; cache_seqlens int32 (B); k_new / v_new None or
// (B, Snew, Hkv, D), written into the cache in place at keys [cache_seqlens[b], + Snew) before the attention.
// Returns out (B, Sq, Hq, D) and lse (B, Hq, Sq).  num_splits as flash_attention_v2_general.
std::vector<torch::Tensor> flash_attention_v2_kvcache(torch::Tensor q, torch::Tensor k_cache, torch::Tensor v_cache,
                                                      torch::Tensor cache_seqlens, std::optional<torch::Tensor> block_table,
                                                      std::optional<torch::Tensor> k_new,
                                                      std::optional<torch::Tensor> v_new, bool is_causal,
                                                      float softmax_scale, int64_t num_splits) {
  KvcacheCall c = check_kvcache(q, k_cache, v_cache, cache_seqlens, block_table, k_new, v_new, num_splits);
  return kvcache_fwd(c, is_causal, softmax_scale, num_splits, nullptr, nullptr);
}

namespace {

// The rotary arguments of a cache call (c checked): the tfa_rotary_args but q_rot.  Throws before any device work.
tfa_rotary_args check_rotary(const KvcacheCall& c, const torch::Tensor& rotary_cos, const torch::Tensor& rotary_sin,
                             bool rotary_interleaved) {
  const torch::Tensor& q = c.q;
  TORCH_CHECK(c.snew > 0, "rotary needs k_new and v_new: it rotates the appended keys");
  TORCH_CHECK(rotary_cos.device() == q.device() && rotary_sin.device() == q.device(),
              "rotary_cos and rotary_sin must be on q's device");
  TORCH_CHECK(rotary_cos.scalar_type() == q.scalar_type() && rotary_sin.scalar_type() == q.scalar_type(),
              "rotary_cos and rotary_sin must have q's dtype");
  TORCH_CHECK(rotary_cos.dim() == 2 && rotary_cos.sizes() == rotary_sin.sizes(),
              "rotary_cos and rotary_sin must both be (seqlen_ro, rotary_dim / 2)");
  TORCH_CHECK(rotary_cos.is_contiguous() && rotary_sin.is_contiguous(), "rotary_cos and rotary_sin must be contiguous");
  const int64_t seqlen_ro = rotary_cos.size(0), rotary_dim = 2 * rotary_cos.size(1);
  TORCH_CHECK(rotary_dim >= 16 && rotary_dim <= c.D && rotary_dim % 16 == 0,
              fmt_msg("rotary_dim (2 * rotary_cos.size(1) = %lld) must be a multiple of 16 in [16, head_dim = %lld]",
                      static_cast<long long>(rotary_dim), static_cast<long long>(c.D)));
  TORCH_CHECK(seqlen_ro < (1LL << 31), "rotary_cos and rotary_sin are too large");
  TORCH_CHECK(seqlen_ro >= c.mbps * c.page,
              fmt_msg("rotary_cos / rotary_sin need a row per cache position: seqlen_ro = %lld < capacity = %lld",
                      static_cast<long long>(seqlen_ro), static_cast<long long>(c.mbps * c.page)));
  tfa_rotary_args r;
  r.cos = rotary_cos.data_ptr(); r.sin = rotary_sin.data_ptr();
  r.seqlen_ro = static_cast<int32_t>(seqlen_ro); r.rotary_dim = static_cast<int32_t>(rotary_dim);
  r.interleaved = rotary_interleaved ? 1 : 0;
  r.q_rot = nullptr;
  return r;
}

// The per-tensor scales of an FP8 cache call; throws before any device work.
tfa_kv_quant_args check_quant(double k_scale, double v_scale) {
  TORCH_CHECK(std::isfinite(k_scale) && k_scale > 0 && std::isfinite(v_scale) && v_scale > 0,
              "k_scale and v_scale must be finite and > 0");
  tfa_kv_quant_args qa;
  qa.cache_dtype = TFA_FP8_E4M3;
  qa.k_scale = static_cast<float>(k_scale);
  qa.v_scale = static_cast<float>(v_scale);
  return qa;
}

}  // namespace

// The same with rotary position embedding (flash-attn's rotary_cos / rotary_sin / rotary_interleaved): q and k_new
// are rotated at their absolute positions (tfa_attn_kvcache_rotary_fwd in include/tfa_b200.h) before the attention;
// the caller's q and k_new are not modified.  rotary_cos / rotary_sin (seqlen_ro, rotary_dim / 2) contiguous in q's
// dtype on q's device, seqlen_ro >= capacity, rotary_dim a multiple of 16 in [16, D]; k_new / v_new are required.
std::vector<torch::Tensor> flash_attention_v2_kvcache_rotary(
    torch::Tensor q, torch::Tensor k_cache, torch::Tensor v_cache, torch::Tensor cache_seqlens,
    std::optional<torch::Tensor> block_table, std::optional<torch::Tensor> k_new, std::optional<torch::Tensor> v_new,
    torch::Tensor rotary_cos, torch::Tensor rotary_sin, bool rotary_interleaved, bool is_causal, float softmax_scale,
    int64_t num_splits) {
  KvcacheCall c = check_kvcache(q, k_cache, v_cache, cache_seqlens, block_table, k_new, v_new, num_splits);
  tfa_rotary_args r = check_rotary(c, rotary_cos, rotary_sin, rotary_interleaved);
  return kvcache_fwd(c, is_causal, softmax_scale, num_splits, &r, nullptr);
}

// flash_attention_v2_kvcache (and, with rotary_cos / rotary_sin, flash_attention_v2_kvcache_rotary) against an FP8
// cache: k_cache / v_cache are float8_e4m3fn, an element x8 standing for k_scale * x8 in K and v_scale * x8 in V;
// k_new / v_new (q's dtype) are quantized into them (tfa_attn_kvcache_fp8_fwd in include/tfa_b200.h).
std::vector<torch::Tensor> flash_attention_v2_kvcache_fp8(
    torch::Tensor q, torch::Tensor k_cache, torch::Tensor v_cache, torch::Tensor cache_seqlens,
    std::optional<torch::Tensor> block_table, std::optional<torch::Tensor> k_new, std::optional<torch::Tensor> v_new,
    double k_scale, double v_scale, bool is_causal, float softmax_scale, int64_t num_splits,
    std::optional<torch::Tensor> rotary_cos, std::optional<torch::Tensor> rotary_sin, bool rotary_interleaved) {
  KvcacheCall c = check_kvcache(q, k_cache, v_cache, cache_seqlens, block_table, k_new, v_new, num_splits, true);
  const tfa_kv_quant_args qa = check_quant(k_scale, v_scale);
  TORCH_CHECK(rotary_cos.has_value() == rotary_sin.has_value(), "rotary_cos and rotary_sin must be given together");
  tfa_rotary_args r;
  if (rotary_cos.has_value()) r = check_rotary(c, *rotary_cos, *rotary_sin, rotary_interleaved);
  return kvcache_fwd(c, is_causal, softmax_scale, num_splits, rotary_cos.has_value() ? &r : nullptr, &qa);
}

// A packed variable-length batch of queries against a (paged) KV cache (flash-attn's flash_attn_varlen_func with
// block_table and seqused_k): q (total_q, Hq, D) with cu_seqlens_q int32 (B + 1) offsets as flash_attention_v2_varlen;
// k_cache / v_cache / block_table / cache_seqlens as flash_attention_v2_kvcache; k_new / v_new None or packed
// (total_q, Hkv, D) sharing cu_seqlens_q, written into the cache in place at keys [cache_seqlens[b], + the sequence's
// query rows) before the attention.  Returns out (total_q, Hq, D) and lse (Hq, total_q).  No split-KV.
namespace {

// flash_attention_v2_varlen_kvcache, or with `quant` its FP8-cache form.
std::vector<torch::Tensor> varlen_kvcache(
    const torch::Tensor& q, const torch::Tensor& k_cache, const torch::Tensor& v_cache,
    const torch::Tensor& cu_seqlens_q, int64_t max_seqlen_q, const torch::Tensor& cache_seqlens,
    const std::optional<torch::Tensor>& block_table, const std::optional<torch::Tensor>& k_new,
    const std::optional<torch::Tensor>& v_new, bool is_causal, float softmax_scale, const tfa_kv_quant_args* quant) {
  TFA_CHECK_CUDA(q);
  TORCH_CHECK(q.dim() == 3, "q must have 3 dimensions (total_q, heads, head_dim)");
  TORCH_CHECK(cu_seqlens_q.scalar_type() == at::kInt, "cu_seqlens_q must be int32");
  TORCH_CHECK(cu_seqlens_q.device() == q.device(), "cu_seqlens_q must be on q's device");
  TORCH_CHECK(cu_seqlens_q.dim() == 1 && cu_seqlens_q.is_contiguous(), "cu_seqlens_q must be a contiguous 1-D tensor");
  TORCH_CHECK(cu_seqlens_q.numel() >= 2, fmt_msg("cu_seqlens_q must hold B + 1 >= 2 offsets, got %lld",
                                                 static_cast<long long>(cu_seqlens_q.numel())));
  const int64_t total_q = q.size(0), Hq = q.size(1), D = q.size(2);
  const int64_t B = cu_seqlens_q.numel() - 1;
  const CacheShape cs = check_cache(q, B, k_cache, v_cache, cache_seqlens, block_table, k_new, v_new, quant != nullptr);
  const int64_t nblk = cs.nblk, page = cs.page, Hkv = cs.Hkv, mbps = cs.mbps, bts = cs.bts;
  if (k_new.has_value()) {
    const torch::Tensor &kn = *k_new, &vn = *v_new;
    TORCH_CHECK(kn.dim() == 3 && kn.sizes() == vn.sizes() && kn.strides() == vn.strides() && kn.size(0) == total_q &&
                    kn.size(1) == Hkv && kn.size(2) == D && kn.stride(2) == 1,
                "k_new and v_new must be (total_q, Hkv, D) with identical strides and a unit head_dim stride");
  }
  TORCH_CHECK(D == 64 || D == 128, fmt_msg("head_dim must be 64 or 128, got %lld", static_cast<long long>(D)));
  TORCH_CHECK(total_q >= 1 && Hq >= 1 && Hkv >= 1, "empty tensors are not supported");
  TORCH_CHECK(Hq % Hkv == 0, fmt_msg("query heads (%lld) must be a multiple of K/V heads (%lld)",
                                     static_cast<long long>(Hq), static_cast<long long>(Hkv)));
  TORCH_CHECK(max_seqlen_q >= 1 && max_seqlen_q <= total_q,
              fmt_msg("max_seqlen_q must be in [1, total_q = %lld], got %lld", static_cast<long long>(total_q),
                      static_cast<long long>(max_seqlen_q)));
  TORCH_CHECK(total_q < (1LL << 31) && B < (1LL << 31) && nblk < (1LL << 31) && page < (1LL << 31) &&
                  mbps < (1LL << 31),
              "tensors too large");

  torch::Tensor out, lse;
  int rc = 0;
  {
    c10::cuda::CUDAGuard guard(q.device());
    out = torch::empty({total_q, Hq, D}, q.options());
    lse = torch::empty({Hq, total_q}, q.options().dtype(at::kFloat));
    tfa_attn_varlen_kvcache_args a;
    std::memset(&a, 0, sizeof(a));
    a.q = q.data_ptr(); a.k_cache = k_cache.data_ptr(); a.v_cache = v_cache.data_ptr();
    a.k_new = k_new.has_value() ? k_new->data_ptr() : nullptr;
    a.v_new = v_new.has_value() ? v_new->data_ptr() : nullptr;
    a.out = out.data_ptr(); a.lse = lse.data_ptr<float>();
    a.cu_seqlens_q = cu_seqlens_q.data_ptr<int32_t>();
    a.cache_seqlens = cache_seqlens.data_ptr<int32_t>();
    a.block_table = block_table.has_value() ? block_table->data_ptr<int32_t>() : nullptr;
    a.B = static_cast<int32_t>(B); a.Hq = static_cast<int32_t>(Hq); a.Hkv = static_cast<int32_t>(Hkv);
    a.D = static_cast<int32_t>(D);
    a.total_q = static_cast<int32_t>(total_q); a.max_seqlen_q = static_cast<int32_t>(max_seqlen_q);
    a.num_blocks = static_cast<int32_t>(nblk); a.page_block_size = static_cast<int32_t>(page);
    a.max_blocks_per_seq = static_cast<int32_t>(mbps);
    a.q_stride_s = q.stride(0); a.q_stride_h = q.stride(1);
    a.cache_stride_block = k_cache.stride(0); a.cache_stride_s = k_cache.stride(1); a.cache_stride_h = k_cache.stride(2);
    a.block_table_stride = bts;
    if (k_new.has_value()) { a.new_stride_s = k_new->stride(0); a.new_stride_h = k_new->stride(1); }
    a.dtype = q.scalar_type() == at::kBFloat16 ? TFA_BF16 : TFA_FP16;
    a.is_causal = is_causal ? 1 : 0;
    a.softmax_scale = softmax_scale;
    a.out_fp32 = 0;
    a.stream = at::cuda::getCurrentCUDAStream(q.device().index()).stream();
    rc = quant ? tfa_attn_varlen_kvcache_fp8_fwd(&a, quant) : tfa_attn_varlen_kvcache_fwd(&a);
  }
  raise_on_error(rc);
  return {out, lse};
}

}  // namespace

std::vector<torch::Tensor> flash_attention_v2_varlen_kvcache(
    torch::Tensor q, torch::Tensor k_cache, torch::Tensor v_cache, torch::Tensor cu_seqlens_q, int64_t max_seqlen_q,
    torch::Tensor cache_seqlens, std::optional<torch::Tensor> block_table, std::optional<torch::Tensor> k_new,
    std::optional<torch::Tensor> v_new, bool is_causal, float softmax_scale) {
  return varlen_kvcache(q, k_cache, v_cache, cu_seqlens_q, max_seqlen_q, cache_seqlens, block_table, k_new, v_new,
                        is_causal, softmax_scale, nullptr);
}

// The same against an FP8 cache (float8_e4m3fn k_cache / v_cache with per-tensor k_scale / v_scale), as
// flash_attention_v2_kvcache_fp8.
std::vector<torch::Tensor> flash_attention_v2_varlen_kvcache_fp8(
    torch::Tensor q, torch::Tensor k_cache, torch::Tensor v_cache, torch::Tensor cu_seqlens_q, int64_t max_seqlen_q,
    torch::Tensor cache_seqlens, std::optional<torch::Tensor> block_table, std::optional<torch::Tensor> k_new,
    std::optional<torch::Tensor> v_new, double k_scale, double v_scale, bool is_causal, float softmax_scale) {
  const tfa_kv_quant_args qa = check_quant(k_scale, v_scale);
  return varlen_kvcache(q, k_cache, v_cache, cu_seqlens_q, max_seqlen_q, cache_seqlens, block_table, k_new, v_new,
                        is_causal, softmax_scale, &qa);
}

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
  m.def("flash_attention_v2_cutlass", &flash_attention_v2_cutlass,
        "Flash attention v2 forward, H100-native (sm_90a wgmma/TMA)");
  // the name BASELINE.json's north_star uses for the same call
  m.def("flash_attn_fwd", &flash_attention_v2_cutlass, "alias of flash_attention_v2_cutlass");
  m.def("flash_attention_v2_bshd", &flash_attention_v2_bshd, "same op on (B,S,H,D) tensors");
  m.def("flash_attention_v2_fp32out", &flash_attention_v2_fp32out, "same op, fp32 output (validation)");
  m.def("flash_attention_v2_general", &flash_attention_v2_general,
        "grouped K/V heads, Sq != Sk (bottom-right causal), optional split-KV: (q, k, v, is_causal, scale, num_splits)");
  m.def("flash_attention_v2_fp8", &flash_attention_v2_fp8,
        "FP8 attention: float8_e4m3fn q, k, v with per-tensor scales, e4m3 tensor cores -> [out (out_dtype), lse]",
        py::arg("q"), py::arg("k"), py::arg("v"), py::arg("q_scale"), py::arg("k_scale"), py::arg("v_scale"),
        py::arg("is_causal"), py::arg("softmax_scale"), py::arg("out_dtype"), py::arg("num_splits") = 1);
  m.def("flash_attention_v2_varlen", &flash_attention_v2_varlen,
        "packed variable-length batch: (q, k, v, cu_seqlens_q, cu_seqlens_k, max_seqlen_q, is_causal, scale)");
  m.def("flash_attention_v2_varlen_fp8", &flash_attention_v2_varlen_fp8,
        "FP8 packed variable-length batch: float8_e4m3fn q, k, v with per-tensor scales, e4m3 tensor cores -> [out "
        "(out_dtype), lse]",
        py::arg("q"), py::arg("k"), py::arg("v"), py::arg("cu_seqlens_q"), py::arg("cu_seqlens_k"),
        py::arg("max_seqlen_q"), py::arg("q_scale"), py::arg("k_scale"), py::arg("v_scale"), py::arg("is_causal"),
        py::arg("softmax_scale"), py::arg("out_dtype"));
  m.def("flash_attention_v2_kvcache", &flash_attention_v2_kvcache,
        "attention against a (paged) KV cache with an optional in-place append: (q, k_cache, v_cache, cache_seqlens, "
        "block_table, k_new, v_new, is_causal, scale, num_splits)");
  m.def("flash_attention_v2_kvcache_rotary", &flash_attention_v2_kvcache_rotary,
        "the KV-cache forward with q and k_new rotated (RoPE) at their cache positions: (q, k_cache, v_cache, "
        "cache_seqlens, block_table, k_new, v_new, rotary_cos, rotary_sin, rotary_interleaved, is_causal, scale, "
        "num_splits)");
  m.def("flash_attention_v2_varlen_kvcache", &flash_attention_v2_varlen_kvcache,
        "a packed variable-length batch of queries against a (paged) KV cache with an optional in-place append: (q, "
        "k_cache, v_cache, cu_seqlens_q, max_seqlen_q, cache_seqlens, block_table, k_new, v_new, is_causal, scale)");
  m.def("flash_attention_v2_kvcache_fp8", &flash_attention_v2_kvcache_fp8,
        "the KV-cache forward against an FP8 (float8_e4m3fn) cache with per-tensor scales, k_new / v_new quantized on "
        "append, optional rotary",
        py::arg("q"), py::arg("k_cache"), py::arg("v_cache"), py::arg("cache_seqlens"), py::arg("block_table"),
        py::arg("k_new"), py::arg("v_new"), py::arg("k_scale"), py::arg("v_scale"), py::arg("is_causal"),
        py::arg("softmax_scale"), py::arg("num_splits"), py::arg("rotary_cos") = py::none(),
        py::arg("rotary_sin") = py::none(), py::arg("rotary_interleaved") = false);
  m.def("flash_attention_v2_varlen_kvcache_fp8", &flash_attention_v2_varlen_kvcache_fp8,
        "a packed variable-length batch of queries against an FP8 (float8_e4m3fn) cache with per-tensor scales: (q, "
        "k_cache, v_cache, cu_seqlens_q, max_seqlen_q, cache_seqlens, block_table, k_new, v_new, k_scale, v_scale, "
        "is_causal, scale)");
  m.def("launch_count",[]() { return tfa_launch_count(); }, "kernels launched by the library so far");
  m.def("abi_version", []() { return tfa_abi_version(); });
}
