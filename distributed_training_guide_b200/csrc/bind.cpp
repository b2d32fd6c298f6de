// Python bindings: torch tensors -> raw-pointer launchers (api.h).  Compiled by g++ only.
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <torch/extension.h>

#include "api.h"
#include "comm_api.h"

namespace {

using torch::Tensor;

inline cudaStream_t stream() { return at::cuda::getCurrentCUDAStream().stream(); }

void check_bf16_2d(const Tensor& t, const char* name) {
  TORCH_CHECK(t.is_cuda(), name, " must be a CUDA tensor");
  TORCH_CHECK(t.scalar_type() == at::kBFloat16, name, " must be bfloat16");
  TORCH_CHECK(t.dim() == 2, name, " must be 2-D");
  TORCH_CHECK(t.stride(1) == 1, name, " must have a contiguous last dimension");
}
void check_contig(const Tensor& t, const char* name, at::ScalarType dt) {
  TORCH_CHECK(t.is_cuda() && t.is_contiguous(), name, " must be a contiguous CUDA tensor");
  TORCH_CHECK(t.scalar_type() == dt, name, " has the wrong dtype");
}
// Operands the kernels read or write in 16-byte vectors: contiguous is not enough, a view may start at any element.
void check_vec(const Tensor& t, const char* name, at::ScalarType dt) {
  check_contig(t, name, dt);
  TORCH_CHECK(reinterpret_cast<uintptr_t>(t.data_ptr()) % 16 == 0, name,
              " must start at a 16-byte aligned address (the kernel accesses it in 16-byte vectors)");
}

void gemm(const Tensor& a, const Tensor& b, Tensor& out, bool trans_a, bool trans_b, bool accumulate, int variant) {
  check_bf16_2d(a, "a");
  check_bf16_2d(b, "b");
  check_bf16_2d(out, "out");
  const c10::cuda::CUDAGuard guard(a.device());
  const int M = (int)(trans_a ? a.size(1) : a.size(0));
  const int K = (int)(trans_a ? a.size(0) : a.size(1));
  const int N = (int)(trans_b ? b.size(0) : b.size(1));
  const int Kb = (int)(trans_b ? b.size(1) : b.size(0));
  TORCH_CHECK(K == Kb, "gemm: inner dimensions differ (", K, " vs ", Kb, ")");
  TORCH_CHECK(out.size(0) == M && out.size(1) == N, "gemm: out has the wrong shape");
  dtg::gemm_bf16(a.data_ptr(), b.data_ptr(), out.data_ptr(), M, N, K, a.stride(0), b.stride(0), out.stride(0),
                 /*a_kmajor=*/!trans_a, /*b_kmajor=*/trans_b, accumulate, variant, stream());
}

void check_fp8_2d(const Tensor& t, const char* name) {
  TORCH_CHECK(t.is_cuda(), name, " must be a CUDA tensor");
  TORCH_CHECK(t.scalar_type() == at::kFloat8_e4m3fn || t.scalar_type() == at::kFloat8_e5m2, name,
              " must be float8_e4m3fn or float8_e5m2");
  TORCH_CHECK(t.dim() == 2, name, " must be 2-D");
  TORCH_CHECK(t.stride(1) == 1, name, " must have a contiguous last dimension");
}
void check_scalar_f32(const Tensor& t, const char* name) {
  TORCH_CHECK(t.is_cuda() && t.scalar_type() == at::kFloat && t.numel() == 1, name,
              " must be a one-element float32 CUDA tensor");
}

// out[M,N] (+)= scale_a * scale_b * a[M,K] @ b[N,K]^T; a e4m3 or e5m2, b e4m3; the scales stay on the device
void gemm_fp8(const Tensor& a, const Tensor& b, Tensor& out, const Tensor& scale_a, const Tensor& scale_b,
              bool accumulate, int variant) {
  check_fp8_2d(a, "a");
  check_fp8_2d(b, "b");
  check_bf16_2d(out, "out");
  TORCH_CHECK(b.scalar_type() == at::kFloat8_e4m3fn, "gemm_fp8: b must be float8_e4m3fn");
  check_scalar_f32(scale_a, "scale_a");
  check_scalar_f32(scale_b, "scale_b");
  const c10::cuda::CUDAGuard guard(a.device());
  const int M = (int)a.size(0), K = (int)a.size(1), N = (int)b.size(0);
  TORCH_CHECK(b.size(1) == K, "gemm_fp8: inner dimensions differ (", K, " vs ", b.size(1), ")");
  TORCH_CHECK(out.size(0) == M && out.size(1) == N, "gemm_fp8: out has the wrong shape");
  dtg::gemm_fp8(a.data_ptr(), b.data_ptr(), out.data_ptr(), M, N, K, a.stride(0), b.stride(0), out.stride(0),
                a.scalar_type() == at::kFloat8_e5m2, scale_a.data_ptr<float>(), scale_b.data_ptr<float>(), accumulate,
                variant, stream());
}

Tensor fp8_amax(const Tensor& x) {
  check_bf16_2d(x, "x");
  const c10::cuda::CUDAGuard guard(x.device());
  Tensor amax = torch::empty({1}, x.options().dtype(at::kFloat));
  dtg::fp8_amax(x.data_ptr(), x.size(0), (int)x.size(1), x.stride(0), amax.data_ptr<float>(), stream());
  return amax;
}

// (x8 [R,C] or None, x8^T [C,R] or None, scale_inv [1]) of a bf16 [R,C] matrix given its device amax
std::tuple<c10::optional<Tensor>, c10::optional<Tensor>, Tensor> fp8_cast_transpose(const Tensor& x, const Tensor& amax,
                                                                                    bool e5m2, bool rowwise,
                                                                                    bool transposed) {
  check_bf16_2d(x, "x");
  check_scalar_f32(amax, "amax");
  TORCH_CHECK(rowwise || transposed, "fp8_cast_transpose: ask for at least one layout");
  TORCH_CHECK(x.numel() > 0, "fp8_cast_transpose: empty tensor");
  const c10::cuda::CUDAGuard guard(x.device());
  const auto dt = e5m2 ? at::kFloat8_e5m2 : at::kFloat8_e4m3fn;
  const int64_t R = x.size(0), C = x.size(1);
  c10::optional<Tensor> out, out_t;
  if (rowwise) out = torch::empty({R, C}, x.options().dtype(dt));
  if (transposed) out_t = torch::empty({C, R}, x.options().dtype(dt));
  Tensor scale_inv = torch::empty({1}, x.options().dtype(at::kFloat));
  dtg::fp8_cast_transpose(x.data_ptr(), x.stride(0), (int)R, (int)C, e5m2, amax.data_ptr<float>(),
                          out ? out->data_ptr() : nullptr, out_t ? out_t->data_ptr() : nullptr,
                          scale_inv.data_ptr<float>(), stream());
  return {out, out_t, scale_inv};
}

std::tuple<Tensor, Tensor, c10::optional<Tensor>> rmsnorm_fwd(const Tensor& x, const Tensor& w, double eps,
                                                              const c10::optional<Tensor>& res) {
  check_vec(x, "x", at::kBFloat16);
  check_vec(w, "w", at::kBFloat16);
  const c10::cuda::CUDAGuard guard(x.device());
  const int T = (int)x.size(0), H = (int)x.size(1);
  TORCH_CHECK(w.numel() == H, "rmsnorm: w must have one entry per column of x");
  Tensor y = torch::empty_like(x);
  Tensor rstd = torch::empty({T}, x.options().dtype(at::kFloat));
  c10::optional<Tensor> h;
  const void* rp = nullptr;
  void* hp = nullptr;
  if (res.has_value()) {
    check_vec(*res, "residual", at::kBFloat16);
    TORCH_CHECK(res->sizes() == x.sizes(), "rmsnorm: residual and x differ in shape");
    h = torch::empty_like(x);
    rp = res->data_ptr();
    hp = h->data_ptr();
  }
  dtg::rmsnorm_fwd(x.data_ptr(), rp, w.data_ptr(), y.data_ptr(), hp, rstd.data_ptr<float>(), T, H, (float)eps,
                   stream());
  return {y, rstd, h};
}

std::tuple<Tensor, Tensor> rmsnorm_bwd(const Tensor& dy, const Tensor& h, const Tensor& w, const Tensor& rstd,
                                       const c10::optional<Tensor>& dres) {
  check_vec(dy, "dy", at::kBFloat16);
  check_vec(h, "h", at::kBFloat16);
  check_vec(w, "w", at::kBFloat16);
  check_contig(rstd, "rstd", at::kFloat);
  const c10::cuda::CUDAGuard guard(dy.device());
  const int T = (int)dy.size(0), H = (int)dy.size(1);
  TORCH_CHECK(h.sizes() == dy.sizes() && w.numel() == H && rstd.numel() == T, "rmsnorm_bwd: shapes differ");
  Tensor dx = torch::empty_like(dy);
  Tensor dw = torch::empty({H}, dy.options().dtype(at::kFloat));
  Tensor partial = torch::empty({dtg::rmsnorm_bwd_grid(T), H}, dy.options().dtype(at::kFloat));
  const void* dr = nullptr;
  if (dres.has_value()) {
    check_vec(*dres, "dres", at::kBFloat16);
    TORCH_CHECK(dres->sizes() == dy.sizes(), "rmsnorm_bwd: dres and dy differ in shape");
    dr = dres->data_ptr();
  }
  dtg::rmsnorm_bwd(dy.data_ptr(), h.data_ptr(), w.data_ptr(), rstd.data_ptr<float>(), dr, dx.data_ptr(),
                   partial.data_ptr<float>(), dw.data_ptr<float>(), T, H, stream());
  return {dx, dw};
}

void rope_inplace(Tensor& qkv, const Tensor& cos, const Tensor& sin, int64_t n_rot, bool inverse) {
  // qkv: [B, S, heads, d] contiguous; cos/sin fp32 [S, d/2] or [B, S, d/2]
  check_vec(qkv, "qkv", at::kBFloat16);
  check_vec(cos, "cos", at::kFloat);
  check_vec(sin, "sin", at::kFloat);
  TORCH_CHECK(qkv.dim() == 4, "qkv must be [B,S,heads,d]");
  const c10::cuda::CUDAGuard guard(qkv.device());
  const int64_t B = qkv.size(0), S = qkv.size(1), NH = qkv.size(2), d = qkv.size(3);
  const bool per_token = cos.dim() == 3;
  TORCH_CHECK(cos.size(-1) == d / 2 && cos.size(per_token ? 1 : 0) == S, "cos/sin table has the wrong shape");
  TORCH_CHECK(sin.sizes() == cos.sizes(), "cos and sin differ in shape");
  TORCH_CHECK(n_rot >= 0 && n_rot <= NH, "rope: n_rot must be within [0, heads]");
  dtg::rope_inplace(qkv.data_ptr(), cos.data_ptr<float>(), sin.data_ptr<float>(), B * S, (int)S, (int)NH, (int)n_rot,
                    (int)d, per_token, inverse, stream());
}

Tensor swiglu_fwd(const Tensor& gu) {
  check_vec(gu, "gu", at::kBFloat16);
  const c10::cuda::CUDAGuard guard(gu.device());
  const int64_t T = gu.size(0), I = gu.size(1) / 2;
  Tensor h = torch::empty({T, I}, gu.options());
  dtg::swiglu_fwd(gu.data_ptr(), h.data_ptr(), T, (int)I, stream());
  return h;
}
Tensor swiglu_bwd(const Tensor& dh, const Tensor& gu) {
  check_vec(dh, "dh", at::kBFloat16);
  check_vec(gu, "gu", at::kBFloat16);
  const c10::cuda::CUDAGuard guard(gu.device());
  Tensor dgu = torch::empty_like(gu);
  dtg::swiglu_bwd(dh.data_ptr(), gu.data_ptr(), dgu.data_ptr(), gu.size(0), (int)(gu.size(1) / 2), stream());
  return dgu;
}

Tensor cross_entropy_fwd_bwd(Tensor& logits, const Tensor& targets) {
  check_vec(logits, "logits", at::kBFloat16);
  check_contig(targets, "targets", at::kLong);
  const c10::cuda::CUDAGuard guard(logits.device());
  const int T = (int)logits.size(0), V = (int)logits.size(1);
  TORCH_CHECK(targets.numel() == T, "targets must have one entry per logits row");
  Tensor scratch = torch::empty({T + 2}, logits.options().dtype(at::kFloat));
  float* sp = scratch.data_ptr<float>();
  dtg::cross_entropy_fwd_bwd(logits.data_ptr(), (const long long*)targets.data_ptr<int64_t>(),
                             sp + 2, sp, sp + 1, T, V, stream());
  return scratch.slice(0, 1, 2).reshape({});
}

void scale_inplace(Tensor& x, const Tensor& scale) {
  check_vec(x, "x", at::kBFloat16);
  check_contig(scale, "scale", at::kFloat);
  const c10::cuda::CUDAGuard guard(x.device());
  dtg::scale_inplace(x.data_ptr(), scale.data_ptr<float>(), x.numel(), stream());
}

Tensor embedding_fwd(const Tensor& ids, const Tensor& w) {
  check_contig(ids, "ids", at::kLong);
  check_vec(w, "w", at::kBFloat16);
  const c10::cuda::CUDAGuard guard(w.device());
  Tensor out = torch::empty({ids.numel(), w.size(1)}, w.options());
  dtg::embedding_fwd((const long long*)ids.data_ptr<int64_t>(), w.data_ptr(), out.data_ptr(), ids.numel(),
                     (int)w.size(1), stream());
  return out;
}
void embedding_bwd_sorted(const Tensor& dout, const Tensor& ids_sorted, const Tensor& perm, Tensor& dw, bool accumulate) {
  check_vec(dout, "dout", at::kBFloat16);
  check_vec(dw, "dw", at::kBFloat16);
  check_contig(ids_sorted, "ids_sorted", at::kLong);
  check_contig(perm, "perm", at::kLong);
  TORCH_CHECK(perm.numel() == ids_sorted.numel(), "int64 ids / permutation");
  const c10::cuda::CUDAGuard guard(dw.device());
  dtg::embedding_bwd_sorted(dout.data_ptr(), (const long long*)ids_sorted.data_ptr<int64_t>(),
                            (const long long*)perm.data_ptr<int64_t>(), dw.data_ptr(), ids_sorted.numel(),
                            (int)dw.size(1), accumulate, at::cuda::getCurrentCUDAStream().stream());
}

// dw (+)= the per-id sum of dout's rows; the [T, H] fp32 scratch and the [V] slot table live until the call returns
// (the caching allocator keeps them on this stream)
void embedding_bwd(const Tensor& dout, const Tensor& ids, Tensor& dw, bool accumulate) {
  check_vec(dout, "dout", at::kBFloat16);
  check_contig(ids, "ids", at::kLong);
  check_vec(dw, "dw", at::kBFloat16);
  TORCH_CHECK(dw.dim() == 2 && dout.dim() == 2 && dout.size(1) == dw.size(1) && dout.size(0) == ids.numel(),
              "embedding_bwd: dout must be [T, H] for T ids and dw [V, H]");
  const c10::cuda::CUDAGuard guard(dw.device());
  const int64_t T = ids.numel(), V = dw.size(0), H = dw.size(1);
  Tensor slot = torch::empty({V}, dw.options().dtype(at::kInt));
  Tensor sums = torch::empty({T, H}, dw.options().dtype(at::kFloat));
  dtg::embedding_bwd(dout.data_ptr(), (const long long*)ids.data_ptr<int64_t>(), dw.data_ptr(),
                     reinterpret_cast<unsigned int*>(slot.data_ptr<int>()), sums.data_ptr<float>(), T, V, (int)H,
                     accumulate, stream());
}

void adamw_flat(Tensor& p, const Tensor& g, Tensor& m, Tensor& v, double lr, double b1, double b2, double eps,
                double wd, int64_t step, double grad_scale) {
  check_vec(p, "p", at::kBFloat16);
  check_vec(g, "g", at::kBFloat16);
  check_vec(m, "exp_avg", m.scalar_type());
  check_vec(v, "exp_avg_sq", v.scalar_type());
  TORCH_CHECK(m.scalar_type() == v.scalar_type(), "exp_avg / exp_avg_sq dtypes differ");
  const bool fp32 = m.scalar_type() == at::kFloat;
  TORCH_CHECK(fp32 || m.scalar_type() == at::kBFloat16, "optimizer state must be bf16 or fp32");
  TORCH_CHECK(p.numel() == g.numel() && p.numel() == m.numel() && p.numel() == v.numel(), "size mismatch");
  const c10::cuda::CUDAGuard guard(p.device());
  dtg::adamw_flat(p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), p.numel(), (float)lr, (float)b1, (float)b2,
                  (float)eps, (float)wd, (int)step, (float)grad_scale, fp32, stream());
}

}  // namespace

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
  m.doc() = "distributed_training_guide_b200 sm_90a kernels";
  m.def("launch_count", []() { return (uint64_t)dtg::launch_count(); });
  m.def("gemm", &gemm, py::arg("a"), py::arg("b"), py::arg("out"), py::arg("trans_a") = false,
        py::arg("trans_b") = false, py::arg("accumulate") = false, py::arg("variant") = 0);
  m.def("gemm_fp8", &gemm_fp8, py::arg("a"), py::arg("b"), py::arg("out"), py::arg("scale_a"), py::arg("scale_b"),
        py::arg("accumulate") = false, py::arg("variant") = 0);
  m.def("fp8_amax", &fp8_amax);
  m.def("fp8_cast_transpose", &fp8_cast_transpose, py::arg("x"), py::arg("amax"), py::arg("e5m2"),
        py::arg("rowwise") = true, py::arg("transposed") = true);
  m.def("gemm_max_active_clusters",[](int cg) { return dtg::gemm_max_active_clusters(cg); });
  m.def("rmsnorm_fwd", &rmsnorm_fwd);
  m.def("rmsnorm_bwd", &rmsnorm_bwd);
  m.def("rope_inplace", &rope_inplace);
  m.def("swiglu_fwd", &swiglu_fwd);
  m.def("swiglu_bwd", &swiglu_bwd);
  m.def("cross_entropy_fwd_bwd", &cross_entropy_fwd_bwd);
  m.def("scale_inplace", &scale_inplace);
  m.def("embedding_fwd", &embedding_fwd);
  m.def("embedding_bwd", &embedding_bwd, py::arg("dout"), py::arg("ids"), py::arg("dw"), py::arg("accumulate") = false);
  m.def("embedding_bwd_sorted", &embedding_bwd_sorted);
  m.def("adamw_flat", &adamw_flat);
  dtg::bind_comm(m);
  dtg::bind_attention(m);
  dtg::bind_tp(m);
  dtg::bind_dataloader(m);
  dtg::bind_symm_vmm(m);
}
