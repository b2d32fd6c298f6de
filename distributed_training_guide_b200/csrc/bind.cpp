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

// A bias [N] for the bias epilogue of the forward GEMMs: every refusal names the argument and happens before a launch.
const void* check_gemm_bias(const c10::optional<Tensor>& bias, const Tensor& out, int64_t N, bool accumulate,
                            bool forward_layout, const char* who) {
  if (!bias.has_value()) return nullptr;
  const Tensor& b = *bias;
  TORCH_CHECK(b.is_cuda() && b.device() == out.device(), who, ": bias must be on the device of out");
  TORCH_CHECK(b.scalar_type() == at::kBFloat16, who, ": bias must be bfloat16");
  TORCH_CHECK(b.dim() == 1 && b.size(0) == N, who, ": bias must be [N] = [", N, "]");
  TORCH_CHECK(b.is_contiguous(), who, ": bias must be contiguous");
  TORCH_CHECK(reinterpret_cast<uintptr_t>(b.data_ptr()) % 16 == 0, who,
              ": bias must start at a 16-byte aligned address");
  TORCH_CHECK(!accumulate, who, ": bias cannot be combined with accumulate=True");
  TORCH_CHECK(forward_layout, who, ": bias needs the forward layout (trans_a unset, trans_b set)");
  return b.data_ptr();
}

void gemm(const Tensor& a, const Tensor& b, Tensor& out, bool trans_a, bool trans_b, bool accumulate, int variant,
          const c10::optional<Tensor>& bias) {
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
  const void* bp = check_gemm_bias(bias, out, N, accumulate, !trans_a && trans_b, "gemm");
  TORCH_CHECK(!bp || K > 0, "gemm: bias needs K >= 1");
  dtg::gemm_bf16(a.data_ptr(), b.data_ptr(), out.data_ptr(), M, N, K, a.stride(0), b.stride(0), out.stride(0),
                 /*a_kmajor=*/!trans_a, /*b_kmajor=*/trans_b, accumulate, variant, stream(), bp);
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
              bool accumulate, int variant, const c10::optional<Tensor>& bias) {
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
  const void* bp = check_gemm_bias(bias, out, N, accumulate, true, "gemm_fp8");
  TORCH_CHECK(!bp || a.scalar_type() == at::kFloat8_e4m3fn, "gemm_fp8: bias needs a float8_e4m3fn a (the forward GEMM)");
  TORCH_CHECK(!bp || K > 0, "gemm_fp8: bias needs K >= 1");
  dtg::gemm_fp8(a.data_ptr(), b.data_ptr(), out.data_ptr(), M, N, K, a.stride(0), b.stride(0), out.stride(0),
                a.scalar_type() == at::kFloat8_e5m2, scale_a.data_ptr<float>(), scale_b.data_ptr<float>(), accumulate,
                variant, stream(), bp);
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

// ---- row norms (norm.cu) ------------------------------------------------------------------------------------------
// Every norm binding validates its arguments with check_norm before it allocates or launches anything, and returns
// empty outputs and zero gradients for T == 0 without a launch.
using Named = std::pair<const Tensor*, const char*>;   // an operand and the name its errors use; null: not given

// x (or dy): bf16 [T, H], contiguous and 16-byte aligned, H a positive multiple of 8 up to the kind's limit.  rows:
// x's shape; params: bf16 [H]; stats: fp32 [T]; all on x's device.  eps, in a forward: finite, > 0 for LayerNorm and
// >= 0 for RMSNorm.  Returns H.
int64_t check_norm(const char* who, dtg::NormKind k, Named x, std::initializer_list<Named> rows,
                   std::initializer_list<Named> params, std::initializer_list<Named> stats, const double* eps) {
  const Tensor& x0 = *x.first;
  check_vec(x0, x.second, at::kBFloat16);
  TORCH_CHECK(x0.dim() == 2, who, ": ", x.second, " must be 2-D [T, H]");
  const int64_t T = x0.size(0), H = x0.size(1), max_h = dtg::norm_max_hidden(k);
  TORCH_CHECK(H > 0 && H % 8 == 0 && H <= max_h, who, ": hidden size must be a positive multiple of 8 and <= ", max_h,
              ", got ", H);
  for (const auto& [t, name] : rows) {
    if (!t) continue;
    check_vec(*t, name, at::kBFloat16);
    TORCH_CHECK(t->sizes() == x0.sizes() && t->device() == x0.device(), who, ": ", name, " and ", x.second,
                " differ in shape or device");
  }
  for (const auto& [t, name] : params) {
    check_vec(*t, name, at::kBFloat16);
    TORCH_CHECK(t->dim() == 1 && t->size(0) == H, who, ": ", name, " must be [H] = [", H, "]");
    TORCH_CHECK(t->device() == x0.device(), who, ": ", name, " must be on the device of ", x.second);
  }
  for (const auto& [t, name] : stats) {
    if (!t) continue;
    check_contig(*t, name, at::kFloat);
    TORCH_CHECK(t->dim() == 1 && t->size(0) == T && t->device() == x0.device(), who, ": ", name, " must be [T] = [", T,
                "] on the device of ", x.second);
  }
  if (eps) {
    const bool ln = k != dtg::NormKind::kRms;
    TORCH_CHECK(std::isfinite(*eps) && (ln ? *eps > 0 : *eps >= 0), who, ": eps must be finite and ",
                ln ? "> 0" : ">= 0", ", got ", *eps);
  }
  return H;
}

c10::optional<Tensor> optional(const Tensor& t) { return t.defined() ? c10::optional<Tensor>(t) : c10::nullopt; }

struct NormOut {
  Tensor y1, y2, h, mean, rstd;   // undefined where the variant has no such output
};

// params: w (RMSNorm), w, b (LayerNorm) or w1, b1, w2, b2 (LayerNorm2); r: the residual, or null
NormOut norm_fwd(const char* who, dtg::NormKind k, dtg::NormRes mode, const Tensor& x, const Tensor* r,
                 const char* rname, std::initializer_list<Named> params, double eps) {
  const int64_t H = check_norm(who, k, {&x, "x"}, {{r, rname}}, params, {}, &eps);
  const c10::cuda::CUDAGuard guard(x.device());
  const int64_t T = x.size(0);
  const bool ln = k != dtg::NormKind::kRms;
  NormOut o;
  if (mode != dtg::NormRes::kAddAfter) o.y1 = torch::empty_like(x);
  if (k == dtg::NormKind::kLn2) o.y2 = torch::empty_like(x);
  if (r) o.h = torch::empty_like(x);
  if (ln) o.mean = torch::empty({T}, x.options().dtype(at::kFloat));
  o.rstd = torch::empty({T}, x.options().dtype(at::kFloat));
  if (T == 0) return o;
  auto ptr = [](const Tensor& t) { return t.defined() ? t.data_ptr() : nullptr; };
  dtg::NormFwdArgs a{};
  a.x = x.data_ptr();
  a.r = r ? r->data_ptr() : nullptr;
  const Named* p = params.begin();
  for (int q = 0; q < (k == dtg::NormKind::kLn2 ? 2 : 1); ++q) {
    a.w[q] = (p++)->first->data_ptr();
    if (ln) a.b[q] = (p++)->first->data_ptr();
  }
  a.y[0] = ptr(o.y1);
  a.y[1] = ptr(o.y2);
  a.h = ptr(o.h);
  a.mean = ln ? o.mean.data_ptr<float>() : nullptr;
  a.rstd = o.rstd.data_ptr<float>();
  dtg::norm_fwd(k, mode, a, (int)T, (int)H, (float)eps, stream());
  return o;
}

// (dx, dparams fp32 [norm_grad_planes(k), H]); dx += dres when dres is given
std::pair<Tensor, Tensor> norm_bwd(const char* who, dtg::NormKind k, const Tensor& dy1, const char* dyname,
                                   const Tensor* dy2, const Tensor& h, std::initializer_list<Named> gains,
                                   const Tensor* mean, const Tensor& rstd, const c10::optional<Tensor>& dres) {
  const Tensor* dr = dres.has_value() ? &*dres : nullptr;
  const int64_t H = check_norm(who, k, {&dy1, dyname}, {{dy2, "dy2"}, {&h, "h"}, {dr, "dres"}}, gains,
                               {{mean, "mean"}, {&rstd, "rstd"}}, nullptr);
  const c10::cuda::CUDAGuard guard(dy1.device());
  const int64_t T = dy1.size(0), planes = dtg::norm_grad_planes(k);
  const auto f32 = dy1.options().dtype(at::kFloat);
  Tensor dx = torch::empty_like(dy1);
  if (T == 0) return {dx, torch::zeros({planes, H}, f32)};
  Tensor dparams = torch::empty({planes, H}, f32);
  Tensor partial = torch::empty({planes, dtg::norm_bwd_grid(k, (int)T, (int)H), H}, f32);
  dtg::NormBwdArgs a{};
  a.dy[0] = dy1.data_ptr();
  a.dy[1] = dy2 ? dy2->data_ptr() : nullptr;
  a.h = h.data_ptr();
  int q = 0;
  for (const auto& g : gains) a.w[q++] = g.first->data_ptr();
  a.mean = mean ? mean->data_ptr<float>() : nullptr;
  a.rstd = rstd.data_ptr<float>();
  a.dres = dr ? dr->data_ptr() : nullptr;
  a.dx = dx.data_ptr();
  a.partial = partial.data_ptr<float>();
  a.dparams = dparams.data_ptr<float>();
  dtg::norm_bwd(k, a, (int)T, (int)H, stream());
  return {dx, dparams};
}

int norm_bwd_grid(dtg::NormKind k, const char* who, int64_t T, int64_t H) {
  TORCH_CHECK(T > 0 && H > 0 && H % 8 == 0 && H <= dtg::norm_max_hidden(k), who, ": bad shape");
  return dtg::norm_bwd_grid(k, (int)T, (int)H);
}

// (y, rstd, h or None): h = bf16(x + residual) when a residual is given, y = RMSNorm(h) * w
std::tuple<Tensor, Tensor, c10::optional<Tensor>> rmsnorm_fwd(const Tensor& x, const Tensor& w, double eps,
                                                              const c10::optional<Tensor>& res) {
  const Tensor* r = res.has_value() ? &*res : nullptr;
  const NormOut o = norm_fwd("rmsnorm_fwd", dtg::NormKind::kRms, r ? dtg::NormRes::kAddBefore : dtg::NormRes::kNone,
                             x, r, "residual", {{&w, "w"}}, eps);
  return {o.y1, o.rstd, optional(o.h)};
}

// (h, rstd) with h = bf16(r + bf16(rmsnorm(x) * w)): the norm-then-add of OLMo 2's post-sublayer norms
std::tuple<Tensor, Tensor> rmsnorm_add_fwd(const Tensor& x, const Tensor& r, const Tensor& w, double eps) {
  const NormOut o = norm_fwd("rmsnorm_add", dtg::NormKind::kRms, dtg::NormRes::kAddAfter, x, &r, "r", {{&w, "w"}}, eps);
  return {o.h, o.rstd};
}

// (dx, dw fp32) of y = RMSNorm(h) * w, with dx += dres when dres is given
std::tuple<Tensor, Tensor> rmsnorm_bwd(const Tensor& dy, const Tensor& h, const Tensor& w, const Tensor& rstd,
                                       const c10::optional<Tensor>& dres) {
  auto [dx, d] = norm_bwd("rmsnorm_bwd", dtg::NormKind::kRms, dy, "dy", nullptr, h, {{&w, "w"}}, nullptr, rstd, dres);
  return {dx, d[0]};
}

// (y, h or None, mean, rstd): h = bf16(x + residual) when a residual is given, y = LayerNorm(h) * w + b
std::tuple<Tensor, c10::optional<Tensor>, Tensor, Tensor> layernorm_fwd(const Tensor& x,
                                                                       const c10::optional<Tensor>& res,
                                                                       const Tensor& w, const Tensor& b, double eps) {
  const Tensor* r = res.has_value() ? &*res : nullptr;
  const NormOut o = norm_fwd("layernorm_fwd", dtg::NormKind::kLn, r ? dtg::NormRes::kAddBefore : dtg::NormRes::kNone,
                             x, r, "residual", {{&w, "w"}, {&b, "b"}}, eps);
  return {o.y1, optional(o.h), o.mean, o.rstd};
}

// (dx, dw fp32, db fp32) of y = LayerNorm(h) * w + b, with dx += dres when dres is given
std::tuple<Tensor, Tensor, Tensor> layernorm_bwd(const Tensor& dy, const Tensor& h, const Tensor& w, const Tensor& mean,
                                                 const Tensor& rstd, const c10::optional<Tensor>& dres) {
  auto [dx, d] = norm_bwd("layernorm_bwd", dtg::NormKind::kLn, dy, "dy", nullptr, h, {{&w, "w"}}, &mean, rstd, dres);
  return {dx, d[0], d[1]};
}

// (y1, y2, h or None, mean, rstd): h = bf16(x + residual) when a residual is given, y_i = LayerNorm(h) * w_i + b_i
std::tuple<Tensor, Tensor, c10::optional<Tensor>, Tensor, Tensor> layernorm2_fwd(
    const Tensor& x, const c10::optional<Tensor>& res, const Tensor& w1, const Tensor& b1, const Tensor& w2,
    const Tensor& b2, double eps) {
  const Tensor* r = res.has_value() ? &*res : nullptr;
  const NormOut o = norm_fwd("layernorm2_fwd", dtg::NormKind::kLn2, r ? dtg::NormRes::kAddBefore : dtg::NormRes::kNone,
                             x, r, "residual", {{&w1, "w1"}, {&b1, "b1"}, {&w2, "w2"}, {&b2, "b2"}}, eps);
  return {o.y1, o.y2, optional(o.h), o.mean, o.rstd};
}

// (dx, dparams fp32 [4, H] = dw1, db1, dw2, db2) of the two LayerNorms, with dx += dres when dres is given
std::tuple<Tensor, Tensor> layernorm2_bwd(const Tensor& dy1, const Tensor& dy2, const Tensor& h, const Tensor& w1,
                                          const Tensor& w2, const Tensor& mean, const Tensor& rstd,
                                          const c10::optional<Tensor>& dres) {
  auto [dx, d] = norm_bwd("layernorm2_bwd", dtg::NormKind::kLn2, dy1, "dy1", &dy2, h, {{&w1, "w1"}, {&w2, "w2"}}, &mean,
                          rstd, dres);
  return {dx, d};
}

Tensor gelu_tanh_fwd(const Tensor& x) {
  check_vec(x, "x", at::kBFloat16);
  TORCH_CHECK(x.numel() % 8 == 0, "gelu_tanh_fwd: x must have a multiple of 8 elements, got ", x.numel());
  const c10::cuda::CUDAGuard guard(x.device());
  Tensor y = torch::empty_like(x);
  if (x.numel() > 0) dtg::gelu_tanh_fwd(x.data_ptr(), y.data_ptr(), x.numel(), stream());
  return y;
}

Tensor gelu_tanh_bwd(const Tensor& dy, const Tensor& x) {
  check_vec(dy, "dy", at::kBFloat16);
  check_vec(x, "x", at::kBFloat16);
  TORCH_CHECK(dy.sizes() == x.sizes() && dy.device() == x.device(), "gelu_tanh_bwd: dy and x differ in shape or device");
  TORCH_CHECK(x.numel() % 8 == 0, "gelu_tanh_bwd: x must have a multiple of 8 elements, got ", x.numel());
  const c10::cuda::CUDAGuard guard(x.device());
  Tensor dx = torch::empty_like(x);
  if (x.numel() > 0) dtg::gelu_tanh_bwd(dy.data_ptr(), x.data_ptr(), dx.data_ptr(), x.numel(), stream());
  return dx;
}

// cos/sin tables of the RoPE kernels, w = rot_dim / 2 floats per row, for qkv [B, S, heads, d]: fp32, 16-byte aligned,
// both [S, w] (row t % S), [T, w] or [B, S, w] (a row per token), on qkv's device.  Returns per_token.
bool check_rope_tables(const Tensor& qkv, const Tensor& cos, const Tensor& sin, int64_t w, const char* who) {
  check_vec(cos, "cos", at::kFloat);
  check_vec(sin, "sin", at::kFloat);
  const int64_t B = qkv.size(0), S = qkv.size(1);
  TORCH_CHECK(sin.sizes() == cos.sizes(), who, ": cos and sin differ in shape");
  TORCH_CHECK((cos.dim() == 2 || cos.dim() == 3) && cos.size(-1) == w, who, ": cos/sin table has the wrong shape: ",
              cos.sizes(), " is not [S, ", w, "], [T, ", w, "] or [B, S, ", w, "]");
  TORCH_CHECK(cos.dim() == 2 || (cos.size(0) == B && cos.size(1) == S), who, ": cos/sin table has the wrong shape: a ",
              "3-D table must be [B, S, ", w, "] = [", B, ", ", S, ", ", w, "], got ", cos.sizes());
  const int64_t rows = cos.dim() == 2 ? cos.size(0) : B * S;
  TORCH_CHECK(rows == S || rows == B * S, who, ": cos/sin table has the wrong shape: its ", rows,
              " rows match neither S = ", S, " nor T = ", B * S);
  TORCH_CHECK(cos.device() == qkv.device() && sin.device() == qkv.device(), who,
              ": cos and sin must be on the device of qkv");
  return rows != S;
}

void rope_inplace(Tensor& qkv, const Tensor& cos, const Tensor& sin, int64_t n_rot, bool inverse,
                  const c10::optional<int64_t>& rot_dim_arg) {
  // qkv: [B, S, heads, d] contiguous; rot_dim defaults to d
  check_vec(qkv, "qkv", at::kBFloat16);
  TORCH_CHECK(qkv.dim() == 4, "qkv must be [B,S,heads,d]");
  const int64_t B = qkv.size(0), S = qkv.size(1), NH = qkv.size(2), d = qkv.size(3);
  const int64_t rot_dim = rot_dim_arg.has_value() ? *rot_dim_arg : d;
  TORCH_CHECK(rot_dim > 0 && rot_dim <= d && rot_dim % 16 == 0,
              "rope: rot_dim must be a positive multiple of 16 and <= head_dim ", d, ", got ", rot_dim);
  const bool per_token = check_rope_tables(qkv, cos, sin, rot_dim / 2, "rope");
  TORCH_CHECK(n_rot >= 0 && n_rot <= NH, "rope: n_rot must be within [0, heads]");
  const c10::cuda::CUDAGuard guard(qkv.device());
  dtg::rope_inplace(qkv.data_ptr(), cos.data_ptr<float>(), sin.data_ptr<float>(), B * S, (int)S, (int)NH, (int)n_rot,
                    (int)d, (int)rot_dim, per_token, inverse, stream());
}

Tensor gelu_fwd(const Tensor& x) {
  check_vec(x, "x", at::kBFloat16);
  TORCH_CHECK(x.numel() % 8 == 0, "gelu_fwd: x must have a multiple of 8 elements, got ", x.numel());
  const c10::cuda::CUDAGuard guard(x.device());
  Tensor y = torch::empty_like(x);
  if (x.numel() > 0) dtg::gelu_fwd(x.data_ptr(), y.data_ptr(), x.numel(), stream());
  return y;
}

Tensor gelu_bwd(const Tensor& dy, const Tensor& x) {
  check_vec(dy, "dy", at::kBFloat16);
  check_vec(x, "x", at::kBFloat16);
  TORCH_CHECK(dy.sizes() == x.sizes() && dy.device() == x.device(), "gelu_bwd: dy and x differ in shape or device");
  TORCH_CHECK(x.numel() % 8 == 0, "gelu_bwd: x must have a multiple of 8 elements, got ", x.numel());
  const c10::cuda::CUDAGuard guard(x.device());
  Tensor dx = torch::empty_like(x);
  if (x.numel() > 0) dtg::gelu_bwd(dy.data_ptr(), x.data_ptr(), dx.data_ptr(), x.numel(), stream());
  return dx;
}

// QK-norm + RoPE, per head (Qwen3: gains [d]) or, with FULL, over each token's whole q and k regions (OLMo 2: gains
// [nh * d] and [nkv * d]).  Every refusal happens before any launch.
template <bool FULL>
bool check_qk_norm_rope(const Tensor& qkv, const Tensor& q_w, const Tensor& k_w, const Tensor& cos, const Tensor& sin,
                        int64_t nh, int64_t nkv) {
  const char* who = FULL ? "qk_norm_full_rope" : "qk_norm_rope";
  check_vec(qkv, "qkv", at::kBFloat16);
  TORCH_CHECK(qkv.dim() == 4, who, ": qkv must be [B, S, heads, d]");
  const int64_t NH = qkv.size(2), d = qkv.size(3);
  TORCH_CHECK(d == 128, who, ": head_dim must be 128, got ", d);
  TORCH_CHECK(nh >= 1 && nkv >= 1 && NH == nh + 2 * nkv, who, ": qkv has ", NH,
              " heads, expected nh + 2 * nkv with nh, nkv >= 1 (nh = ", nh, ", nkv = ", nkv, ")");
  if (FULL)
    TORCH_CHECK(nh + nkv <= dtg::qk_norm_full_rope_max_heads(), who, ": nh + nkv = ", nh + nkv, " exceeds the ",
                dtg::qk_norm_full_rope_max_heads(), " q + k heads per token the kernel holds");
  check_vec(q_w, "q_w", at::kBFloat16);
  check_vec(k_w, "k_w", at::kBFloat16);
  const int64_t qn = FULL ? nh * d : d, kn = FULL ? nkv * d : d;
  TORCH_CHECK(q_w.dim() == 1 && q_w.size(0) == qn, who, ": q_w must be [", qn, "]");
  TORCH_CHECK(k_w.dim() == 1 && k_w.size(0) == kn, who, ": k_w must be [", kn, "]");
  TORCH_CHECK(q_w.device() == qkv.device() && k_w.device() == qkv.device(), who,
              ": q_w and k_w must be on the device of qkv");
  return check_rope_tables(qkv, cos, sin, d / 2, who);
}

// returns x_save [B, S, nh + nkv, 128] and rstd: [B, S, nh + nkv] per head, [B, S, 2] (q, k) with FULL
template <bool FULL>
std::tuple<Tensor, Tensor> qk_norm_rope_fwd(Tensor& qkv, const Tensor& q_w, const Tensor& k_w, const Tensor& cos,
                                            const Tensor& sin, int64_t nh, int64_t nkv, double eps) {
  const bool per_token = check_qk_norm_rope<FULL>(qkv, q_w, k_w, cos, sin, nh, nkv);
  TORCH_CHECK(std::isfinite(eps) && eps >= 0, FULL ? "qk_norm_full_rope" : "qk_norm_rope",
              ": eps must be finite and >= 0");
  const c10::cuda::CUDAGuard guard(qkv.device());
  const int64_t B = qkv.size(0), S = qkv.size(1);
  Tensor x_save = torch::empty({B, S, nh + nkv, 128}, qkv.options());
  Tensor rstd = torch::empty({B, S, FULL ? 2 : nh + nkv}, qkv.options().dtype(at::kFloat));
  (FULL ? dtg::qk_norm_full_rope_fwd : dtg::qk_norm_rope_fwd)(
      qkv.data_ptr(), q_w.data_ptr(), k_w.data_ptr(), cos.data_ptr<float>(), sin.data_ptr<float>(), x_save.data_ptr(),
      rstd.data_ptr<float>(), B * S, (int)S, (int)qkv.size(2), (int)nh, (int)nkv, per_token, (float)eps, stream());
  return {x_save, rstd};
}

// in place on dqkv's q|k heads; returns dw: [2, 128] (q, k) per head, [(nh + nkv) * 128] with FULL
template <bool FULL>
Tensor qk_norm_rope_bwd(Tensor& dqkv, const Tensor& x_save, const Tensor& rstd, const Tensor& q_w, const Tensor& k_w,
                        const Tensor& cos, const Tensor& sin, int64_t nh, int64_t nkv) {
  const bool per_token = check_qk_norm_rope<FULL>(dqkv, q_w, k_w, cos, sin, nh, nkv);
  const char* who = FULL ? "qk_norm_full_rope_bwd" : "qk_norm_rope_bwd";
  const int64_t B = dqkv.size(0), S = dqkv.size(1), T = B * S, nqk = nh + nkv;
  check_vec(x_save, "x_save", at::kBFloat16);
  check_contig(rstd, "rstd", at::kFloat);
  TORCH_CHECK(x_save.sizes() == at::IntArrayRef({B, S, nqk, 128}) && x_save.device() == dqkv.device(), who,
              ": x_save must be [B, S, nh + nkv, 128] on the device of dqkv");
  TORCH_CHECK(rstd.sizes() == at::IntArrayRef({B, S, FULL ? 2 : nqk}) && rstd.device() == dqkv.device(), who,
              ": rstd must be [B, S, ", FULL ? "2" : "nh + nkv", "] on the device of dqkv");
  const c10::cuda::CUDAGuard guard(dqkv.device());
  Tensor dw = FULL ? torch::empty({nqk * 128}, dqkv.options().dtype(at::kFloat))
                   : torch::empty({2, 128}, dqkv.options().dtype(at::kFloat));
  const int grid = (FULL ? dtg::qk_norm_full_rope_bwd_grid : dtg::qk_norm_rope_bwd_grid)(T, (int)nqk);
  Tensor partial = torch::empty({grid, dw.numel()}, dqkv.options().dtype(at::kFloat));
  (FULL ? dtg::qk_norm_full_rope_bwd : dtg::qk_norm_rope_bwd)(
      dqkv.data_ptr(), x_save.data_ptr(), rstd.data_ptr<float>(), q_w.data_ptr(), k_w.data_ptr(),
      cos.data_ptr<float>(), sin.data_ptr<float>(), partial.data_ptr<float>(), dw.data_ptr<float>(), T, (int)S,
      (int)dqkv.size(2), (int)nh, (int)nkv, per_token, stream());
  return dw;
}

// db[N] fp32 = the column sums of dy [T, N] (bf16, contiguous last dimension), in a fixed order (no atomics)
Tensor bias_grad(const Tensor& dy) {
  TORCH_CHECK(dy.is_cuda(), "bias_grad: dy must be a CUDA tensor");
  TORCH_CHECK(dy.scalar_type() == at::kBFloat16, "bias_grad: dy must be bfloat16");
  TORCH_CHECK(dy.dim() == 2, "bias_grad: dy must be 2-D [T, N]");
  TORCH_CHECK(dy.stride(1) == 1, "bias_grad: dy must have a contiguous last dimension");
  const int64_t T = dy.size(0), N = dy.size(1);
  TORCH_CHECK(N % 8 == 0 && N > 0, "bias_grad: N must be a positive multiple of 8, got ", N);
  TORCH_CHECK(T >= 1, "bias_grad: dy must have at least one row");
  TORCH_CHECK(dy.stride(0) % 8 == 0 && reinterpret_cast<uintptr_t>(dy.data_ptr()) % 16 == 0,
              "bias_grad: dy must start at a 16-byte aligned address with a row stride that is a multiple of 8");
  const c10::cuda::CUDAGuard guard(dy.device());
  Tensor db = torch::empty({N}, dy.options().dtype(at::kFloat));
  Tensor partial = torch::empty({dtg::bias_grad_chunks(T, (int)N), N}, dy.options().dtype(at::kFloat));
  dtg::bias_grad(dy.data_ptr(), T, (int)N, dy.stride(0), partial.data_ptr<float>(), db.data_ptr<float>(), stream());
  return db;
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
  dtg::check_loss_args(logits, targets, "cross_entropy");
  const c10::cuda::CUDAGuard guard(logits.device());
  const int T = (int)logits.size(0), V = (int)logits.size(1);
  if (T == 0) return torch::zeros({}, logits.options().dtype(at::kFloat));   // as with every target ignored
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
  dtg::check_embedding_args(ids, w, "w", "embedding_fwd");
  const c10::cuda::CUDAGuard guard(w.device());
  Tensor out = torch::empty({ids.numel(), w.size(1)}, w.options());
  dtg::embedding_fwd((const long long*)ids.data_ptr<int64_t>(), w.data_ptr(), out.data_ptr(), ids.numel(), w.size(0),
                     (int)w.size(1), stream());
  return out;
}
void embedding_bwd_sorted(const Tensor& dout, const Tensor& ids_sorted, const Tensor& perm, Tensor& dw, bool accumulate) {
  check_vec(dout, "dout", at::kBFloat16);
  dtg::check_embedding_args(ids_sorted, dw, "dw", "embedding_bwd_sorted");
  check_contig(perm, "perm", at::kLong);
  TORCH_CHECK(perm.numel() == ids_sorted.numel(), "int64 ids / permutation");
  TORCH_CHECK(dout.dim() == 2 && dout.size(0) == ids_sorted.numel() && dout.size(1) == dw.size(1),
              "embedding_bwd_sorted: dout must be [T, H] for T ids and dw [V, H]");
  const c10::cuda::CUDAGuard guard(dw.device());
  dtg::embedding_bwd_sorted(dout.data_ptr(), (const long long*)ids_sorted.data_ptr<int64_t>(),
                            (const long long*)perm.data_ptr<int64_t>(), dw.data_ptr(), ids_sorted.numel(), dw.size(0),
                            (int)dw.size(1), accumulate, at::cuda::getCurrentCUDAStream().stream());
}

// dw (+)= the per-id sum of dout's rows; the [T, H] fp32 scratch and the [V] slot table live until the call returns
// (the caching allocator keeps them on this stream)
void embedding_bwd(const Tensor& dout, const Tensor& ids, Tensor& dw, bool accumulate) {
  check_vec(dout, "dout", at::kBFloat16);
  dtg::check_embedding_args(ids, dw, "dw", "embedding_bwd");
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

namespace dtg {
void check_loss_args(const Tensor& logits, const Tensor& targets, const char* who) {
  check_vec(logits, "logits", at::kBFloat16);
  TORCH_CHECK(logits.dim() == 2, who, ": logits must be 2-D [T, V]");
  TORCH_CHECK(logits.size(1) > 0 && logits.size(1) % 8 == 0, who, ": the vocabulary (logits.size(1)) must be a ",
              "positive multiple of 8, got ", logits.size(1));
  TORCH_CHECK(targets.is_cuda() && targets.device() == logits.device(), who, ": targets must be on logits' device");
  TORCH_CHECK(targets.scalar_type() == at::kLong, who, ": targets must be int64");
  TORCH_CHECK(targets.is_contiguous(), who, ": targets must be contiguous");
  TORCH_CHECK(targets.numel() == logits.size(0), who, ": targets must have one entry per logits row (",
              logits.size(0), "), got ", targets.numel());
}
void check_embedding_args(const Tensor& ids, const Tensor& table, const char* table_name, const char* who) {
  check_vec(table, table_name, at::kBFloat16);
  TORCH_CHECK(table.dim() == 2 && table.size(1) % 8 == 0, who, ": ", table_name,
              " must be 2-D [V, H] with H a multiple of 8");
  TORCH_CHECK(ids.is_cuda() && ids.device() == table.device(), who, ": ids must be on the device of ", table_name);
  TORCH_CHECK(ids.scalar_type() == at::kLong, who, ": ids must be int64");
  TORCH_CHECK(ids.is_contiguous(), who, ": ids must be contiguous");
}
}  // namespace dtg

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
  m.doc() = "distributed_training_guide_b200 sm_90a kernels";
  m.def("launch_count", []() { return (uint64_t)dtg::launch_count(); });
  m.def("gemm", &gemm, py::arg("a"), py::arg("b"), py::arg("out"), py::arg("trans_a") = false,
        py::arg("trans_b") = false, py::arg("accumulate") = false, py::arg("variant") = 0,
        py::arg("bias") = py::none());
  m.def("gemm_fp8", &gemm_fp8, py::arg("a"), py::arg("b"), py::arg("out"), py::arg("scale_a"), py::arg("scale_b"),
        py::arg("accumulate") = false, py::arg("variant") = 0, py::arg("bias") = py::none());
  m.def("bias_grad", &bias_grad, py::arg("dy"));
  m.def("fp8_amax", &fp8_amax);
  m.def("fp8_cast_transpose", &fp8_cast_transpose, py::arg("x"), py::arg("amax"), py::arg("e5m2"),
        py::arg("rowwise") = true, py::arg("transposed") = true);
  m.def("gemm_max_active_clusters",[](int cg) { return dtg::gemm_max_active_clusters(cg); });
  m.def("rmsnorm_fwd", &rmsnorm_fwd);
  m.def("rmsnorm_bwd", &rmsnorm_bwd);
  m.def("rope_inplace", &rope_inplace, py::arg("qkv"), py::arg("cos"), py::arg("sin"), py::arg("n_rot"),
        py::arg("inverse"), py::arg("rot_dim") = py::none());
  m.def("qk_norm_rope_fwd", &qk_norm_rope_fwd<false>);
  m.def("qk_norm_rope_bwd", &qk_norm_rope_bwd<false>);
  m.def("rmsnorm_add_fwd", &rmsnorm_add_fwd);
  m.def("qk_norm_full_rope_fwd", &qk_norm_rope_fwd<true>);
  m.def("qk_norm_full_rope_bwd", &qk_norm_rope_bwd<true>);
  m.def("qk_norm_full_rope_bwd_grid", [](int64_t T, int64_t nqk) {
    TORCH_CHECK(T > 0 && nqk >= 2 && nqk <= dtg::qk_norm_full_rope_max_heads(), "qk_norm_full_rope_bwd_grid: bad shape");
    return dtg::qk_norm_full_rope_bwd_grid(T, (int)nqk);
  });
  m.def("layernorm_fwd", &layernorm_fwd, py::arg("x"), py::arg("residual"), py::arg("w"), py::arg("b"),
        py::arg("eps"));
  m.def("layernorm_bwd", &layernorm_bwd, py::arg("dy"), py::arg("h"), py::arg("w"), py::arg("mean"),
        py::arg("rstd"), py::arg("dres") = py::none());
  m.def("layernorm_bwd_grid",
        [](int64_t T, int64_t H) { return norm_bwd_grid(dtg::NormKind::kLn, "layernorm_bwd_grid", T, H); });
  m.def("gelu_tanh_fwd", &gelu_tanh_fwd, py::arg("x"));
  m.def("gelu_tanh_bwd", &gelu_tanh_bwd, py::arg("dy"), py::arg("x"));
  m.def("gelu_fwd", &gelu_fwd, py::arg("x"));
  m.def("gelu_bwd", &gelu_bwd, py::arg("dy"), py::arg("x"));
  m.def("layernorm2_fwd", &layernorm2_fwd, py::arg("x"), py::arg("residual"), py::arg("w1"), py::arg("b1"),
        py::arg("w2"), py::arg("b2"), py::arg("eps"));
  m.def("layernorm2_bwd", &layernorm2_bwd, py::arg("dy1"), py::arg("dy2"), py::arg("h"), py::arg("w1"),
        py::arg("w2"), py::arg("mean"), py::arg("rstd"), py::arg("dres") = py::none());
  m.def("layernorm2_bwd_grid",
        [](int64_t T, int64_t H) { return norm_bwd_grid(dtg::NormKind::kLn2, "layernorm2_bwd_grid", T, H); });
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
  dtg::bind_moe(m);
}
