// Python bindings for the wgmma flash-attention kernels.
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <torch/extension.h>

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstdlib>
#include <limits>

#include "api.h"
#include "comm_api.h"

namespace dtg {
namespace {
using torch::Tensor;

// Every argument is checked here, before the first launch: a bad head count divides by zero (host and device) or
// reads the wrong heads, and a bad scale turns every output into NaN.
void check_heads_scale(int64_t nh, int64_t nkv, double scale) {
  TORCH_CHECK(nh >= 1 && nkv >= 1, "nh and nkv must be >= 1, got nh ", nh, ", nkv ", nkv);
  TORCH_CHECK(nh % nkv == 0, "nh must be a multiple of nkv, got nh ", nh, ", nkv ", nkv);
  // the kernels take the scale as fp32: it must stay finite and > 0 after that conversion
  const float s = (float)scale;
  TORCH_CHECK(std::isfinite(s) && s > 0.f, "scale must be finite and > 0, got ", scale);
}

bool aligned16(const Tensor& t) { return reinterpret_cast<uintptr_t>(t.data_ptr()) % 16 == 0; }

// head_dim is an argument, never read off the tensors: a qkv whose last dimension disagrees with it is refused
void check_head_dim(int64_t head_dim) {
  TORCH_CHECK(head_dim == 64 || head_dim == 128, "head_dim must be 64 or 128, got ", head_dim);
}

void check_qkv(const Tensor& qkv, int64_t nh, int64_t nkv, double scale, int64_t head_dim) {
  check_heads_scale(nh, nkv, scale);
  check_head_dim(head_dim);
  TORCH_CHECK(qkv.is_cuda() && qkv.is_contiguous() && qkv.scalar_type() == at::kBFloat16,
              "qkv must be a contiguous bf16 CUDA tensor");
  TORCH_CHECK(qkv.dim() == 4 && qkv.size(2) == nh + 2 * nkv && qkv.size(3) == head_dim,
              "qkv must be [B, S, nh+2*nkv, ", head_dim, "]");
  TORCH_CHECK(qkv.size(0) >= 1 && qkv.size(1) >= 128 && qkv.size(1) % 128 == 0,
              "qkv must have B >= 1 and a sequence length S that is a positive multiple of 128, got ", qkv.sizes());
  TORCH_CHECK(aligned16(qkv), "qkv must start on a 16-byte boundary");
}

// o and d_o of the backward: bf16, contiguous, [B, S, nh, head_dim] on the device of qkv, 16-byte aligned
void check_rows(const Tensor& t, const char* name, const Tensor& qkv, int64_t nh, int64_t head_dim) {
  TORCH_CHECK(t.scalar_type() == at::kBFloat16 && t.is_contiguous(), name, " must be a contiguous bf16 tensor");
  TORCH_CHECK(t.dim() == 4 && t.size(0) == qkv.size(0) && t.size(1) == qkv.size(1) && t.size(2) == nh &&
                  t.size(3) == head_dim,
              name, " must be [B, S, nh, ", head_dim, "] = [", qkv.size(0), ", ", qkv.size(1), ", ", nh, ", ",
              head_dim, "], got ", t.sizes());
  TORCH_CHECK(t.device() == qkv.device(), name, " must be on the device of qkv");
  TORCH_CHECK(aligned16(t), name, " must start on a 16-byte boundary");
}

void check_lse(const Tensor& lse, const Tensor& qkv, int64_t nh) {
  TORCH_CHECK(lse.scalar_type() == at::kFloat && lse.is_contiguous(), "lse must be a contiguous fp32 tensor");
  TORCH_CHECK(lse.dim() == 3 && lse.size(0) == qkv.size(0) && lse.size(1) == nh && lse.size(2) == qkv.size(1),
              "lse must be [B, nh, S] = [", qkv.size(0), ", ", nh, ", ", qkv.size(1), "], got ", lse.sizes());
  TORCH_CHECK(lse.device() == qkv.device(), "lse must be on the device of qkv");
}

// doc_start (document masking): int32 [B, S] on the device of qkv, contiguous; None = plain causal attention.
// Any content is safe to pass: the kernels clamp every block index they derive from it.
const int* doc_start_ptr(const c10::optional<Tensor>& doc_start, const Tensor& qkv) {
  if (!doc_start.has_value() || !doc_start->defined()) return nullptr;
  const Tensor& d = *doc_start;
  TORCH_CHECK(d.scalar_type() == at::kInt, "doc_start must be int32");
  TORCH_CHECK(d.dim() == 2 && d.size(0) == qkv.size(0) && d.size(1) == qkv.size(1), "doc_start must be [B, S] = [",
              qkv.size(0), ", ", qkv.size(1), "], got ", d.sizes());
  TORCH_CHECK(d.is_contiguous(), "doc_start must be contiguous");
  TORCH_CHECK(d.device() == qkv.device(), "doc_start must be on the device of qkv");
  return d.data_ptr<int>();
}

// window (sliding-window attention): None = no window, else an int >= 1; refused before any launch otherwise.
// The kernels take 0 for no window.
int window_arg(const c10::optional<int64_t>& window) {
  if (!window.has_value()) return 0;
  TORCH_CHECK(*window >= 1, "window must be an int >= 1 or None, got ", *window);
  return (int)std::min<int64_t>(*window, std::numeric_limits<int>::max());
}

// version: 0 = default (DTG_ATTN_FWD env, else 2), 1 = P through shared memory, 2 = P kept in registers
// (both in attention_fwd.cu)
int default_fwd_version() {
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("DTG_ATTN_FWD");
    v = e ? atoi(e) : 2;
    if (v != 1 && v != 2) v = 2;
  }
  return v;
}

std::tuple<Tensor, Tensor> py_attn_fwd(const Tensor& qkv, int64_t nh, int64_t nkv, double scale, int64_t version,
                                       const c10::optional<Tensor>& doc_start, const c10::optional<int64_t>& window,
                                       int64_t head_dim) {
  check_qkv(qkv, nh, nkv, scale, head_dim);
  TORCH_CHECK(version >= 0 && version <= 2, "version must be 0 (default), 1 or 2, got ", version);
  const int* ds = doc_start_ptr(doc_start, qkv);
  const int win = window_arg(window);
  const c10::cuda::CUDAGuard guard(qkv.device());
  const int64_t B = qkv.size(0), S = qkv.size(1);
  Tensor o = torch::empty({B, S, nh, head_dim}, qkv.options());
  Tensor lse = torch::empty({B, nh, S}, qkv.options().dtype(at::kFloat));
  if (version == 0) version = default_fwd_version();
  auto fn = version == 1 ? dtg::attn_fwd : dtg::attn_fwd2;
  fn(qkv.data_ptr(), o.data_ptr(), lse.data_ptr<float>(), (int)B, (int)S, (int)nh, (int)nkv, (float)scale,
     at::cuda::getCurrentCUDAStream().stream(), ds, win, (int)head_dim);
  return {o, lse};
}

Tensor py_attn_bwd(const Tensor& d_o, const Tensor& qkv, const Tensor& o, const Tensor& lse, int64_t nh, int64_t nkv,
                   double scale, const c10::optional<Tensor>& trace, int64_t mode,
                   const c10::optional<Tensor>& doc_start, const c10::optional<int64_t>& window, int64_t head_dim) {
  check_qkv(qkv, nh, nkv, scale, head_dim);
  TORCH_CHECK(mode >= 0 && mode <= 2, "mode must be 0 (default), 1 or 2, got ", mode);
  const int* ds = doc_start_ptr(doc_start, qkv);
  const int win = window_arg(window);
  check_rows(o, "o", qkv, nh, head_dim);
  check_rows(d_o, "d_o", qkv, nh, head_dim);
  check_lse(lse, qkv, nh);
  float* tr = nullptr;
  if (trace.has_value() && trace->defined()) {
    TORCH_CHECK(trace->scalar_type() == at::kLong && trace->numel() >= 1024 && trace->is_contiguous() &&
                    trace->device() == qkv.device(),
                "trace must be a contiguous int64[1024] on the device of qkv");
    tr = reinterpret_cast<float*>(trace->data_ptr<int64_t>());
  }
  const c10::cuda::CUDAGuard guard(qkv.device());
  const int64_t B = qkv.size(0), S = qkv.size(1);
  Tensor dqkv = torch::empty_like(qkv);
  Tensor delta = torch::empty({B, nh, S}, qkv.options().dtype(at::kFloat));
  dtg::attn_bwd(qkv.data_ptr(), o.data_ptr(), d_o.data_ptr(), lse.data_ptr<float>(), delta.data_ptr<float>(), tr,
                dqkv.data_ptr(), (int)B, (int)S, (int)nh, (int)nkv, (float)scale, (int)mode,
                at::cuda::getCurrentCUDAStream().stream(), ds, win, (int)head_dim);
  return dqkv;
}
}  // namespace

void bind_attention(pybind11::module_& m) {
  m.def("attn_fwd", &py_attn_fwd, pybind11::arg("qkv"), pybind11::arg("nh"), pybind11::arg("nkv"), pybind11::arg("scale"),
        pybind11::arg("version") = 0, pybind11::arg("doc_start") = pybind11::none(),
        pybind11::arg("window") = pybind11::none(), pybind11::arg("head_dim") = 128);
  m.def("attn_bwd", &py_attn_bwd, pybind11::arg("d_o"), pybind11::arg("qkv"), pybind11::arg("o"), pybind11::arg("lse"),
        pybind11::arg("nh"), pybind11::arg("nkv"), pybind11::arg("scale"), pybind11::arg("trace") = pybind11::none(),
        pybind11::arg("mode") = 0,   // 0 = default (DTG_ATTN_BWD), 1 = P/dS through shared memory, 2 = P/dS in registers
        pybind11::arg("doc_start") = pybind11::none(), pybind11::arg("window") = pybind11::none(),
        pybind11::arg("head_dim") = 128);   // 64 or 128; qkv, o and d_o must have it as their last dimension
}
}  // namespace dtg
