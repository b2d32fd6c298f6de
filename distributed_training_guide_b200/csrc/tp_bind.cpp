// Python bindings of the tensor-parallel kernels (distributed GEMM modes, partial-sum reduce,
// vocab-parallel cross entropy, hidden-parallel embedding).
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <pybind11/stl.h>
#include <torch/extension.h>

#include "api.h"
#include "comm.cuh"
#include "comm_api.h"

namespace dtg {
namespace {
using torch::Tensor;
inline cudaStream_t stream() { return at::cuda::getCurrentCUDAStream().stream(); }

// bias [N] of the all-gather / gather GEMMs' forward (b_kmajor) form: each refusal names the argument
const void* check_bias(const c10::optional<Tensor>& bias, const Tensor& out, bool b_kmajor, const char* who) {
  if (!bias.has_value()) return nullptr;
  const Tensor& b = *bias;
  const int64_t N = out.size(1);
  TORCH_CHECK(b.is_cuda() && b.device() == out.device(), who, ": bias must be on the device of out");
  TORCH_CHECK(b.scalar_type() == at::kBFloat16, who, ": bias must be bfloat16");
  TORCH_CHECK(b.dim() == 1 && b.size(0) == N, who, ": bias must be [N] = [", N, "]");
  TORCH_CHECK(b.is_contiguous(), who, ": bias must be contiguous");
  TORCH_CHECK(reinterpret_cast<uintptr_t>(b.data_ptr()) % 16 == 0, who,
              ": bias must start at a 16-byte aligned address");
  TORCH_CHECK(b_kmajor, who, ": bias needs the forward layout (b_kmajor set)");
  return b.data_ptr();
}

SymmPtrs plain(const std::vector<uint64_t>& ptrs) {
  SymmPtrs s{};
  TORCH_CHECK(ptrs.size() >= 1 && ptrs.size() <= (size_t)kMaxRanks, "1..8 ranks supported");
  for (size_t k = 0; k < ptrs.size(); ++k) s.ptr[k] = (char*)ptrs[k];
  return s;
}

void py_gemm_dist(int64_t mode, const std::vector<uint64_t>& a_ptrs, const std::vector<uint64_t>& b_ptrs,
                  const std::vector<uint64_t>& c_ptrs, int64_t M, int64_t N, int64_t K, int64_t lda, int64_t ldb,
                  int64_t ldc, bool b_kmajor, bool accumulate, int64_t nranks, int64_t rank, int64_t rows_per_peer) {
  const void* as[kMaxRanks] = {nullptr};
  const void* bs[kMaxRanks] = {nullptr};
  void* cs[kMaxRanks] = {nullptr};
  for (size_t i = 0; i < a_ptrs.size() && i < (size_t)kMaxRanks; ++i) as[i] = (const void*)a_ptrs[i];
  for (size_t i = 0; i < b_ptrs.size() && i < (size_t)kMaxRanks; ++i) bs[i] = (const void*)b_ptrs[i];
  for (size_t i = 0; i < c_ptrs.size() && i < (size_t)kMaxRanks; ++i) cs[i] = (void*)c_ptrs[i];
  if (mode != 2) {  // local C: replicate so dist.c_ptr[0] is valid
    for (int i = 1; i < kMaxRanks; ++i) cs[i] = cs[0];
  }
  dtg::gemm_bf16_dist((int)mode, as, bs, cs, (int)M, (int)N, (int)K, lda, ldb, ldc, b_kmajor, accumulate, (int)nranks,
                      (int)rank, (int)rows_per_peer, stream());
}

void py_gemm_ag(const std::vector<uint64_t>& a_bufs, const Tensor& b, Tensor& out, bool b_kmajor, int64_t rank,
                int64_t rows_per_peer, Tensor& flags, int64_t ag_epoch, const std::vector<uint64_t>& pads,
                int64_t bar_epoch, int64_t n_comm, const c10::optional<Tensor>& bias) {
  TORCH_CHECK(b.is_cuda() && b.scalar_type() == at::kBFloat16 && b.dim() == 2 && b.stride(1) == 1, "bad B");
  TORCH_CHECK(out.is_cuda() && out.scalar_type() == at::kBFloat16 && out.dim() == 2 && out.stride(1) == 1, "bad out");
  TORCH_CHECK(flags.scalar_type() == at::kInt && flags.is_cuda(), "flags must be an int32 CUDA tensor");
  const void* bp = check_bias(bias, out, b_kmajor, "gemm_ag");
  const c10::cuda::CUDAGuard guard(out.device());
  const int nr = (int)a_bufs.size();
  const int M = (int)out.size(0), N = (int)out.size(1);
  const int K = (int)(b_kmajor ? b.size(1) : b.size(0));
  TORCH_CHECK((b_kmajor ? b.size(0) : b.size(1)) == N, "B does not match out");
  TORCH_CHECK(flags.numel() * 256 >= M, "flags too small");
  const void* as[kMaxRanks] = {nullptr};
  uint32_t* pd[kMaxRanks] = {nullptr};
  for (int i = 0; i < nr; ++i) {
    as[i] = (const void*)a_bufs[i];
    pd[i] = (uint32_t*)pads[i];
  }
  dtg::gemm_bf16_ag(as, b.data_ptr(), out.data_ptr(), M, N, K, b.stride(0), out.stride(0), b_kmajor, nr, (int)rank,
                    (int)rows_per_peer, (uint32_t*)flags.data_ptr<int>(), (uint32_t)ag_epoch, pd, (uint32_t)bar_epoch,
                    (int)n_comm, stream(), bp);
}

// C = a @ op(B) with B = a weight inside the flat buffer `full` (element offset w_off, w_numel elements), gathered
// from the ranks' shards by the kernel itself (FSDP unshard fused into the consuming GEMM)
void py_gemm_bgather(const Tensor& a, Tensor& full, Tensor& out, bool b_kmajor, int64_t b_rows, int64_t b_cols,
                     const std::vector<uint64_t>& shards, int64_t per_numel, int64_t w_off, int64_t w_numel,
                     Tensor& counters, int64_t target, int64_t chunk_shift, const std::vector<uint64_t>& pads,
                     int64_t rank, int64_t bar_epoch, const c10::optional<Tensor>& bias) {
  TORCH_CHECK(a.is_cuda() && a.scalar_type() == at::kBFloat16 && a.dim() == 2 && a.stride(1) == 1, "bad A");
  TORCH_CHECK(out.is_cuda() && out.scalar_type() == at::kBFloat16 && out.dim() == 2 && out.stride(1) == 1, "bad out");
  const void* bp = check_bias(bias, out, b_kmajor, "gemm_bgather");
  TORCH_CHECK(full.is_contiguous() && full.scalar_type() == at::kBFloat16, "full must be the flat bf16 buffer");
  TORCH_CHECK(counters.scalar_type() == at::kInt && counters.is_cuda(), "counters must be an int32 CUDA tensor");
  TORCH_CHECK(w_off + w_numel <= full.numel() && b_rows * b_cols <= w_numel, "weight outside the flat buffer");
  TORCH_CHECK(((int64_t)full.numel() * 2) >> chunk_shift <= counters.numel(), "counter array too small");
  const c10::cuda::CUDAGuard guard(out.device());
  const int nr = (int)shards.size();
  TORCH_CHECK(nr == (int)pads.size() && nr <= kMaxRanks, "shards / pads per rank");
  const int M = (int)out.size(0), N = (int)out.size(1);
  const int K = (int)a.size(1);
  TORCH_CHECK(a.size(0) == M && (b_kmajor ? (b_rows == N && b_cols == K) : (b_rows == K && b_cols == N)),
              "shape mismatch");
  const void* sh[kMaxRanks] = {nullptr};
  uint32_t* pd[kMaxRanks] = {nullptr};
  for (int i = 0; i < nr; ++i) {
    sh[i] = (const void*)shards[i];
    pd[i] = (uint32_t*)pads[i];
  }
  dtg::gemm_bf16_bgather(a.data_ptr(), full.data_ptr(), out.data_ptr(), M, N, K, a.stride(0), b_cols, out.stride(0),
                         b_kmajor, sh, per_numel * 2, w_off * 2, w_numel * 2, (uint32_t*)counters.data_ptr<int>(),
                         (uint32_t)target, (int)chunk_shift, pd, nr, (int)rank, (uint32_t)bar_epoch, stream(), bp);
}

void py_reduce_parts(const Tensor& parts, const c10::optional<Tensor>& residual, Tensor& out) {
  TORCH_CHECK(parts.is_contiguous() && out.is_contiguous() && parts.scalar_type() == at::kBFloat16, "bad tensors");
  const int64_t nparts = parts.size(0);
  TORCH_CHECK(parts.numel() == nparts * out.numel(), "parts must be [nparts, *out.shape]");
  const c10::cuda::CUDAGuard guard(out.device());
  dtg::tp_reduce_parts(parts.data_ptr(), residual.has_value() ? residual->data_ptr() : nullptr, out.data_ptr(),
                       out.numel(), (int)nparts, stream());
}

void py_reduce_mc(uint64_t part_mc, const c10::optional<Tensor>& residual, Tensor& out, const std::vector<uint64_t>& pads,
                  int64_t rank, int64_t epoch, const c10::optional<Tensor>& err) {
  TORCH_CHECK(out.is_contiguous() && out.scalar_type() == at::kBFloat16, "bad out");
  TORCH_CHECK(!residual.has_value() || (residual->is_contiguous() && residual->numel() == out.numel()), "bad residual");
  const c10::cuda::CUDAGuard guard(out.device());
  SymmPads pd{};
  TORCH_CHECK(pads.size() <= (size_t)kMaxRanks, "1..8 ranks supported");
  for (size_t k = 0; k < pads.size(); ++k) pd.ptr[k] = (uint32_t*)pads[k];
  dtg::tp_reduce_mc((const void*)part_mc, residual.has_value() ? residual->data_ptr() : nullptr, out.data_ptr(),
                    out.numel(), pd, (int)rank, (int)pads.size(), (uint32_t)epoch,
                    err.has_value() ? err->data_ptr<int>() : nullptr, stream());
}

void py_vp_ce_stats(const Tensor& logits, const Tensor& targets, Tensor& stats, int64_t v0) {
  TORCH_CHECK(logits.is_contiguous() && logits.scalar_type() == at::kBFloat16 && stats.scalar_type() == at::kFloat, "bad");
  const c10::cuda::CUDAGuard guard(logits.device());
  dtg::vp_ce_stats(logits.data_ptr(), (const long long*)targets.data_ptr<int64_t>(), stats.data_ptr(), (int)logits.size(0),
                   (int)logits.size(1), (int)v0, stream());
}

Tensor py_vp_ce_grad(Tensor& logits, const Tensor& targets, const std::vector<uint64_t>& stats_ptrs, int64_t v0) {
  const c10::cuda::CUDAGuard guard(logits.device());
  const int T = (int)logits.size(0);
  Tensor scratch = torch::empty({T + 2}, logits.options().dtype(at::kFloat));
  float* sp = scratch.data_ptr<float>();
  const long long* tg = (const long long*)targets.data_ptr<int64_t>();
  dtg::ce_count_valid(tg, sp, T, stream());
  dtg::vp_ce_grad(logits.data_ptr(), tg, plain(stats_ptrs), sp + 2, sp, T, (int)logits.size(1), (int)v0,
                  (int)stats_ptrs.size(), stream());
  dtg::ce_finalize(sp + 2, sp, sp + 1, T, stream());
  return scratch.slice(0, 1, 2).reshape({});
}

void py_embed_fwd(const Tensor& ids, const Tensor& w, const std::vector<uint64_t>& dst_ptrs, int64_t rpp, int64_t H,
                  int64_t rank) {
  const c10::cuda::CUDAGuard guard(w.device());
  dtg::tp_embed_fwd((const long long*)ids.data_ptr<int64_t>(), w.data_ptr(), plain(dst_ptrs), ids.numel(), (int)rpp,
                    (int)H, (int)w.size(1), (int)rank, stream());
}
void py_embed_bwd(const Tensor& ids, const std::vector<uint64_t>& dx_ptrs, Tensor& dw, int64_t rpp, int64_t H,
                  int64_t rank) {
  const c10::cuda::CUDAGuard guard(dw.device());
  dtg::tp_embed_bwd((const long long*)ids.data_ptr<int64_t>(), plain(dx_ptrs), dw.data_ptr(), ids.numel(), (int)rpp,
                    (int)H, (int)dw.size(1), (int)rank, stream());
}
}  // namespace

void bind_tp(pybind11::module_& m) {
  m.def("gemm_dist", &py_gemm_dist);
  m.def("gemm_ag", &py_gemm_ag, py::arg("a_bufs"), py::arg("b"), py::arg("out"), py::arg("b_kmajor"), py::arg("rank"),
        py::arg("rows_per_peer"), py::arg("flags"), py::arg("ag_epoch"), py::arg("pads"), py::arg("bar_epoch"),
        py::arg("n_comm"), py::arg("bias") = py::none());
  m.def("gemm_bgather", &py_gemm_bgather, py::arg("a"), py::arg("full"), py::arg("out"), py::arg("b_kmajor"),
        py::arg("b_rows"), py::arg("b_cols"), py::arg("shards"), py::arg("per_numel"), py::arg("w_off"),
        py::arg("w_numel"), py::arg("counters"), py::arg("target"), py::arg("chunk_shift"), py::arg("pads"),
        py::arg("rank"), py::arg("bar_epoch"), py::arg("bias") = py::none());
  m.def("tp_reduce_parts", &py_reduce_parts);
  m.def("tp_reduce_mc", &py_reduce_mc);
  m.def("vp_ce_stats", &py_vp_ce_stats);
  m.def("vp_ce_grad", &py_vp_ce_grad);
  m.def("tp_embed_fwd", &py_embed_fwd);
  m.def("tp_embed_bwd", &py_embed_bwd);
}
}  // namespace dtg
