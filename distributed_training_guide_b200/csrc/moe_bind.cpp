// Python bindings of the mixture-of-experts kernels (moe.cu) and the grouped GEMM.  Every argument is checked here,
// before any launch.
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <torch/extension.h>

#include "api.h"
#include "comm_api.h"

namespace {

using torch::Tensor;

inline cudaStream_t stream() { return at::cuda::getCurrentCUDAStream().stream(); }

void check_t(const Tensor& t, const Tensor& like, at::ScalarType dt, int64_t dim, const char* who, const char* name) {
  TORCH_CHECK(t.is_cuda() && t.device() == like.device(), who, ": ", name, " must be on the device of the other tensors");
  TORCH_CHECK(t.scalar_type() == dt, who, ": ", name, " must be ", c10::toString(dt), ", got ",
              c10::toString(t.scalar_type()));
  TORCH_CHECK(t.dim() == dim, who, ": ", name, " must be ", dim, "-D, got ", t.dim(), "-D");
  TORCH_CHECK(t.is_contiguous(), who, ": ", name, " must be contiguous");
  TORCH_CHECK(reinterpret_cast<uintptr_t>(t.data_ptr()) % 16 == 0, who, ": ", name,
              " must start at a 16-byte aligned address");
}

// seg int32 [E + 1] on x's device; returns E
int64_t check_seg(const Tensor& seg, const Tensor& like, const char* who) {
  check_t(seg, like, at::kInt, 1, who, "seg");
  const int64_t E = seg.size(0) - 1;
  TORCH_CHECK(E >= 1 && E <= dtg::kMoeMaxExperts, who, ": seg must hold E + 1 entries with 1 <= E <= ",
              dtg::kMoeMaxExperts);
  return E;
}

// norm_topk: each token's w row is its top-k probabilities divided by their sum (Qwen3-MoE's norm_topk_prob)
std::tuple<Tensor, Tensor, Tensor, Tensor, Tensor, Tensor, Tensor, Tensor> moe_route(const Tensor& logits, int64_t k,
                                                                                     bool norm_topk) {
  const char* who = "moe_route";
  TORCH_CHECK(logits.is_cuda() && logits.scalar_type() == at::kBFloat16 && logits.dim() == 2 && logits.stride(1) == 1,
              who, ": logits must be a bf16 CUDA [T, E] tensor with a contiguous last dimension");
  const int64_t T = logits.size(0), E = logits.size(1);
  TORCH_CHECK(E >= 1 && E <= dtg::kMoeMaxExperts, who, ": E must be in [1, ", dtg::kMoeMaxExperts, "], got ", E);
  TORCH_CHECK(k >= 1 && k <= E, who, ": k must be in [1, E = ", E, "], got ", k);
  TORCH_CHECK(T * k + E * 128 < (int64_t)INT32_MAX, who, ": too many tokens for int32 row indices");
  const c10::cuda::CUDAGuard guard(logits.device());
  const auto i32 = logits.options().dtype(at::kInt), f32 = logits.options().dtype(at::kFloat);
  const int64_t rows_cap = dtg::moe_rows_cap(T, (int)E, (int)k);
  Tensor p = torch::empty({T, E}, f32), idx = torch::empty({T, k}, i32), w = torch::empty({T, k}, f32);
  Tensor pos = torch::empty({T, k}, i32), seg = torch::empty({E + 1}, i32);
  Tensor tile_expert = torch::empty({rows_cap / 128}, i32), row_tok = torch::empty({rows_cap}, i32);
  Tensor counts = torch::empty({E}, i32);
  Tensor scratch = torch::empty({std::max<int64_t>(dtg::moe_route_scratch(T, (int)E), 1)}, i32);
  if (T == 0) {
    seg.zero_();
    counts.zero_();
    tile_expert.fill_(-1);
    return {p, idx, w, pos, seg, tile_expert, row_tok, counts};
  }
  dtg::moe_route(logits.data_ptr(), logits.stride(0), (int)T, (int)E, (int)k, norm_topk, p.data_ptr<float>(),
                 idx.data_ptr<int>(), w.data_ptr<float>(), pos.data_ptr<int>(), seg.data_ptr<int>(), tile_expert.data_ptr<int>(),
                 row_tok.data_ptr<int>(), counts.data_ptr<int>(), scratch.data_ptr<int>(), stream());
  return {p, idx, w, pos, seg, tile_expert, row_tok, counts};
}

Tensor moe_permute(const Tensor& x, const Tensor& row_tok, const Tensor& seg, int64_t k) {
  const char* who = "moe_permute";
  check_t(x, x, at::kBFloat16, 2, who, "x");
  check_t(row_tok, x, at::kInt, 1, who, "row_tok");
  const int64_t E = check_seg(seg, x, who), T = x.size(0), H = x.size(1);
  TORCH_CHECK(H > 0 && H % 8 == 0, who, ": H must be a positive multiple of 8, got ", H);
  TORCH_CHECK(k >= 1 && k <= E, who, ": k must be in [1, E]");
  const int64_t rows_cap = dtg::moe_rows_cap(T, (int)E, (int)k);
  TORCH_CHECK(row_tok.size(0) == rows_cap, who, ": row_tok must have rows_cap = ", rows_cap, " entries");
  const c10::cuda::CUDAGuard guard(x.device());
  Tensor out = torch::empty({rows_cap, H}, x.options());
  dtg::moe_permute(x.data_ptr(), (int)T, row_tok.data_ptr<int>(), seg.data_ptr<int>(), (int)E, (int)k, (int)H,
                   rows_cap, out.data_ptr(), stream());
  return out;
}

Tensor moe_combine(const Tensor& yp, const Tensor& pos, const c10::optional<Tensor>& w) {
  const char* who = "moe_combine";
  check_t(yp, yp, at::kBFloat16, 2, who, "yp");
  check_t(pos, yp, at::kInt, 2, who, "pos");
  const int64_t T = pos.size(0), k = pos.size(1), H = yp.size(1);
  TORCH_CHECK(H > 0 && H % 8 == 0, who, ": H must be a positive multiple of 8, got ", H);
  TORCH_CHECK(k >= 1, who, ": pos must be [T, k] with k >= 1");
  TORCH_CHECK(T == 0 || yp.size(0) >= 1, who, ": yp has no rows for pos to name");
  if (w.has_value()) {
    check_t(*w, yp, at::kFloat, 2, who, "w");
    TORCH_CHECK(w->size(0) == T && w->size(1) == k, who, ": w must be [T, k] like pos");
  }
  const c10::cuda::CUDAGuard guard(yp.device());
  Tensor out = torch::empty({T, H}, yp.options());
  dtg::moe_combine(yp.data_ptr(), yp.size(0), pos.data_ptr<int>(), w.has_value() ? w->data_ptr<float>() : nullptr,
                   (int)T, (int)k, (int)H, out.data_ptr(), stream());
  return out;
}

std::tuple<Tensor, Tensor> moe_combine_bwd(const Tensor& dy, const Tensor& yp, const Tensor& row_tok, const Tensor& seg,
                                           const Tensor& w) {
  const char* who = "moe_combine_bwd";
  check_t(dy, dy, at::kBFloat16, 2, who, "dy");
  check_t(yp, dy, at::kBFloat16, 2, who, "yp");
  check_t(row_tok, dy, at::kInt, 1, who, "row_tok");
  check_t(w, dy, at::kFloat, 2, who, "w");
  const int64_t E = check_seg(seg, dy, who), T = dy.size(0), H = dy.size(1), k = w.size(1);
  TORCH_CHECK(H > 0 && H % 8 == 0, who, ": H must be a positive multiple of 8, got ", H);
  TORCH_CHECK(w.size(0) == T && k >= 1 && k <= E, who, ": w must be [T, k] with 1 <= k <= E");
  const int64_t rows_cap = dtg::moe_rows_cap(T, (int)E, (int)k);
  TORCH_CHECK(yp.size(0) == rows_cap && yp.size(1) == H, who, ": yp must be [rows_cap, H] = [", rows_cap, ", ", H, "]");
  TORCH_CHECK(row_tok.size(0) == rows_cap, who, ": row_tok must have rows_cap = ", rows_cap, " entries");
  const c10::cuda::CUDAGuard guard(dy.device());
  Tensor dyp = torch::empty({rows_cap, H}, dy.options());
  Tensor dw = torch::empty({T, k}, w.options());
  dtg::moe_combine_bwd(dy.data_ptr(), (int)T, yp.data_ptr(), row_tok.data_ptr<int>(), seg.data_ptr<int>(),
                       w.data_ptr<float>(), (int)E, (int)k, (int)H, rows_cap, dyp.data_ptr(), dw.data_ptr<float>(),
                       stream());
  return {dyp, dw};
}

// norm_topk: the backward of the renormalised weights moe_route(..., norm_topk=True) wrote
Tensor moe_router_bwd(const Tensor& p, const Tensor& idx, const Tensor& dw, const c10::optional<Tensor>& dpsum,
                      bool norm_topk) {
  const char* who = "moe_router_bwd";
  check_t(p, p, at::kFloat, 2, who, "p");
  check_t(idx, p, at::kInt, 2, who, "idx");
  check_t(dw, p, at::kFloat, 2, who, "dw");
  const int64_t T = p.size(0), E = p.size(1), k = idx.size(1);
  TORCH_CHECK(E >= 1 && E <= dtg::kMoeMaxExperts, who, ": E must be in [1, ", dtg::kMoeMaxExperts, "]");
  TORCH_CHECK(idx.size(0) == T && k >= 1 && k <= E, who, ": idx must be [T, k] with 1 <= k <= E");
  TORCH_CHECK(dw.size(0) == T && dw.size(1) == k, who, ": dw must be [T, k] like idx");
  if (dpsum.has_value()) {
    check_t(*dpsum, p, at::kFloat, 1, who, "dpsum");
    TORCH_CHECK(dpsum->size(0) == E, who, ": dpsum must be [E]");
  }
  const c10::cuda::CUDAGuard guard(p.device());
  Tensor dlogits = torch::empty({T, E}, p.options().dtype(at::kBFloat16));
  dtg::moe_router_bwd(p.data_ptr<float>(), idx.data_ptr<int>(), dw.data_ptr<float>(),
                      dpsum.has_value() ? dpsum->data_ptr<float>() : nullptr, (int)T, (int)E, (int)k, norm_topk,
                      dlogits.data_ptr(), stream());
  return dlogits;
}

// fp32 [E] column sums of the router probabilities p [T, E], in a fixed order (the aux loss's P_e, times T)
Tensor moe_prob_sums(const Tensor& p) {
  check_t(p, p, at::kFloat, 2, "moe_prob_sums", "p");
  const c10::cuda::CUDAGuard guard(p.device());
  Tensor out = torch::zeros({p.size(1)}, p.options());
  if (p.size(0) > 0 && p.size(1) > 0) dtg::colsum(p.data_ptr<float>(), out.data_ptr<float>(), (int)p.size(0), (int)p.size(1), stream());
  return out;
}

// mode 0: out [R, N] = a [R, K] . w[e] [N, K]^T;  mode 1: out [R, N] = a [R, K] . w[e] [K, N];  with w [E, ., .] and e
// the expert of a's row tile.  mode 2: out[e] [M, N] (+)= a[seg_e] [., M]^T . b[seg_e] [., N], out [E, M, N].
void gemm_grouped(int64_t mode, const Tensor& a, const Tensor& b, Tensor& out, const Tensor& seg,
                  const c10::optional<Tensor>& tile_expert, bool accumulate) {
  const char* who = "gemm_grouped";
  TORCH_CHECK(mode >= 0 && mode <= 2, who, ": mode must be 0 (forward), 1 (dgrad) or 2 (wgrad)");
  check_t(a, a, at::kBFloat16, 2, who, "a");
  check_t(b, a, at::kBFloat16, mode == 2 ? 2 : 3, who, "b");
  check_t(out, a, at::kBFloat16, mode == 2 ? 3 : 2, who, "out");
  const int64_t E = check_seg(seg, a, who), R = a.size(0);
  int64_t M, N, K;
  if (mode == 2) {
    TORCH_CHECK(b.size(0) == R, who, ": a and b must have the same rows");
    M = a.size(1), N = b.size(1), K = R;
    TORCH_CHECK(out.size(0) == E && out.size(1) == M && out.size(2) == N, who, ": out must be [E, M, N] = [", E, ", ",
                M, ", ", N, "]");
  } else {
    TORCH_CHECK(tile_expert.has_value(), who, ": the forward and dgrad modes need tile_expert");
    check_t(*tile_expert, a, at::kInt, 1, who, "tile_expert");
    TORCH_CHECK(tile_expert->size(0) * 128 == R, who, ": tile_expert must have rows / 128 entries");
    TORCH_CHECK(b.size(0) == E, who, ": b must hold one slab per expert, [E, ., .] with E = ", E);
    K = a.size(1);
    N = mode == 0 ? b.size(1) : b.size(2);
    TORCH_CHECK((mode == 0 ? b.size(2) : b.size(1)) == K, who, ": inner dimensions differ");
    TORCH_CHECK(out.size(0) == R && out.size(1) == N, who, ": out must be [R, N] = [", R, ", ", N, "]");
    M = R;
  }
  TORCH_CHECK(!accumulate || mode == 2, who, ": only the wgrad mode accumulates");
  const c10::cuda::CUDAGuard guard(a.device());
  dtg::gemm_bf16_grouped((int)mode, a.data_ptr(), b.data_ptr(), out.data_ptr(), (int)M, (int)N, (int)K, a.stride(0),
                         mode == 2 ? b.stride(0) : b.stride(1), mode == 2 ? out.stride(1) : out.stride(0), (int)E,
                         seg.data_ptr<int>(), mode == 2 ? nullptr : tile_expert->data_ptr<int>(), accumulate, stream());
}

}  // namespace

namespace dtg {
void bind_moe(pybind11::module_& m) {
  m.def("moe_route", &::moe_route, pybind11::arg("logits"), pybind11::arg("k"), pybind11::arg("norm_topk") = false);
  m.def("moe_permute", &::moe_permute, pybind11::arg("x"), pybind11::arg("row_tok"), pybind11::arg("seg"),
        pybind11::arg("k"));
  m.def("moe_combine", &::moe_combine, pybind11::arg("yp"), pybind11::arg("pos"), pybind11::arg("w") = pybind11::none());
  m.def("moe_combine_bwd", &::moe_combine_bwd, pybind11::arg("dy"), pybind11::arg("yp"), pybind11::arg("row_tok"),
        pybind11::arg("seg"), pybind11::arg("w"));
  m.def("moe_router_bwd", &::moe_router_bwd, pybind11::arg("p"), pybind11::arg("idx"), pybind11::arg("dw"),
        pybind11::arg("dpsum") = pybind11::none(), pybind11::arg("norm_topk") = false);
  m.def("gemm_grouped", &::gemm_grouped, pybind11::arg("mode"), pybind11::arg("a"), pybind11::arg("b"),
        pybind11::arg("out"), pybind11::arg("seg"), pybind11::arg("tile_expert") = pybind11::none(),
        pybind11::arg("accumulate") = false);
  m.def("moe_prob_sums", &::moe_prob_sums, pybind11::arg("p"));
  m.def("moe_rows_cap", [](int64_t T, int64_t E, int64_t k) { return dtg::moe_rows_cap(T, (int)E, (int)k); });
}
}  // namespace dtg
