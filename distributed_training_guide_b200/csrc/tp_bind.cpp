// Python bindings of the tensor-parallel kernels (distributed GEMM modes, partial-sum reduce,
// vocab-parallel cross entropy, hidden-parallel embedding).
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <pybind11/stl.h>
#include <torch/extension.h>

#include <tuple>

#include "api.h"
#include "comm.cuh"
#include "comm_api.h"

namespace dtg {
namespace {
using torch::Tensor;
inline cudaStream_t stream() { return at::cuda::getCurrentCUDAStream().stream(); }

// bias [N] of the all-gather GEMM's forward (b_kmajor) form: each refusal names the argument
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

// ---- distributed GEMMs and the partial-sum reduce ----------------------------------------------------------------
// gemm_dist, gemm_ag and tp_reduce_parts validate their arguments with check_dist before anything is
// launched.  The kernels index their peer-pointer arrays by rank and owner, so a list of the wrong length or a rank
// out of range would read or write through a pointer nobody passed.
using PeerList = std::tuple<const std::vector<uint64_t>*, const char*, int64_t>;   // list, name, entries read
struct Operand {
  const Tensor* t;   // null: not given
  const char* name;
  at::ScalarType dtype;
  bool flat;         // contiguous; otherwise 2-D with a contiguous last dimension (a row-strided matrix)
};

// nranks in 1..8 and 0 <= rank < nranks; every list exactly as long as the kernel reads it, each entry a nonzero
// 16-byte aligned address (TMA bases, bulk copies and 16-byte vectors); every operand on `dev`'s device (the current
// device when dev is null), of its dtype and layout, 16-byte aligned.
void check_dist(const char* who, std::initializer_list<PeerList> lists, int64_t nranks, int64_t rank, const Tensor* dev,
                std::initializer_list<Operand> ops) {
  TORCH_CHECK(nranks >= 1 && nranks <= kMaxRanks, who, ": 1..", kMaxRanks, " ranks, got ", nranks);
  TORCH_CHECK(rank >= 0 && rank < nranks, who, ": rank ", rank, " outside the ", nranks, " ranks");
  for (const auto& [v, name, want] : lists) {
    TORCH_CHECK((int64_t)v->size() == want, who, ": ", name, " must have ", want, " entries, got ", v->size());
    for (uint64_t p : *v)
      TORCH_CHECK(p != 0 && p % 16 == 0, who, ": every entry of ", name, " must be a 16-byte aligned address");
  }
  const c10::Device d = dev ? dev->device() : c10::Device(c10::kCUDA, c10::cuda::current_device());
  for (const auto& o : ops) {
    if (!o.t) continue;
    const Tensor& t = *o.t;
    TORCH_CHECK(t.is_cuda() && t.device() == d, who, ": ", o.name, " must be on ", d);
    TORCH_CHECK(t.scalar_type() == o.dtype, who, ": ", o.name, " must be ", c10::toString(o.dtype));
    if (o.flat) {
      TORCH_CHECK(t.is_contiguous(), who, ": ", o.name, " must be contiguous");
    } else {
      TORCH_CHECK(t.dim() == 2 && t.stride(1) == 1, who, ": ", o.name, " must be 2-D with a contiguous last dimension");
    }
    TORCH_CHECK(reinterpret_cast<uintptr_t>(t.data_ptr()) % 16 == 0, who, ": ", o.name,
                " must start at a 16-byte aligned address");
  }
}

// mode 1 reads nranks A bases, mode 3 nranks B bases, mode 4 nranks A bases, mode 2 writes nranks C bases (each
// already offset to this rank's slot); every other list has one entry.  Mode 2 always overwrites its slots.
void py_gemm_dist(int64_t mode, const std::vector<uint64_t>& a_ptrs, const std::vector<uint64_t>& b_ptrs,
                  const std::vector<uint64_t>& c_ptrs, int64_t M, int64_t N, int64_t K, int64_t lda, int64_t ldb,
                  int64_t ldc, bool b_kmajor, bool accumulate, int64_t nranks, int64_t rank, int64_t rows_per_peer) {
  TORCH_CHECK(mode >= 1 && mode <= 4, "gemm_dist: mode must be 1..4, got ", mode);
  const int64_t na = (mode == 1 || mode == 4) ? nranks : 1, nb = mode == 3 ? nranks : 1, nc = mode == 2 ? nranks : 1;
  check_dist("gemm_dist", {{&a_ptrs, "a_ptrs", na}, {&b_ptrs, "b_ptrs", nb}, {&c_ptrs, "c_ptrs", nc}}, nranks, rank,
             nullptr, {});
  TORCH_CHECK(M >= 0 && N >= 0 && K >= 0 && rows_per_peer >= 0, "gemm_dist: negative extent");
  TORCH_CHECK(mode != 2 || !accumulate, "gemm_dist: mode 2 overwrites the staging slots (accumulate is not supported)");
  const void* as[kMaxRanks] = {nullptr};
  const void* bs[kMaxRanks] = {nullptr};
  void* cs[kMaxRanks] = {nullptr};
  for (int64_t i = 0; i < na; ++i) as[i] = (const void*)a_ptrs[i];
  for (int64_t i = 0; i < nb; ++i) bs[i] = (const void*)b_ptrs[i];
  for (int64_t i = 0; i < nc; ++i) cs[i] = (void*)c_ptrs[i];
  dtg::gemm_bf16_dist((int)mode, as, bs, cs, (int)M, (int)N, (int)K, lda, ldb, ldc, b_kmajor, accumulate, (int)nranks,
                      (int)rank, (int)rows_per_peer, stream());
}

// a_bufs and pads: one entry per rank.  The kernel waits for ag_epoch on the tile flags and for bar_epoch on the
// signal pads, so with more than one rank neither may be 0 (the waits would pass before anything arrived).
void py_gemm_ag(const std::vector<uint64_t>& a_bufs, const Tensor& b, Tensor& out, bool b_kmajor, int64_t rank,
                int64_t rows_per_peer, Tensor& flags, int64_t ag_epoch, const std::vector<uint64_t>& pads,
                int64_t bar_epoch, int64_t n_comm, const c10::optional<Tensor>& bias) {
  const int64_t nr = (int64_t)a_bufs.size();
  check_dist("gemm_ag", {{&a_bufs, "a_bufs", nr}, {&pads, "pads", nr}}, nr, rank, &out,
             {{&b, "b", at::kBFloat16, false}, {&out, "out", at::kBFloat16, false}, {&flags, "flags", at::kInt, true}});
  const void* bp = check_bias(bias, out, b_kmajor, "gemm_ag");
  TORCH_CHECK(nr == 1 || ((uint32_t)ag_epoch != 0 && (uint32_t)bar_epoch != 0),
              "gemm_ag: ag_epoch and bar_epoch must be nonzero with more than one rank");
  const c10::cuda::CUDAGuard guard(out.device());
  const int M = (int)out.size(0), N = (int)out.size(1);
  const int K = (int)(b_kmajor ? b.size(1) : b.size(0));
  TORCH_CHECK((b_kmajor ? b.size(0) : b.size(1)) == N, "gemm_ag: B does not match out");
  TORCH_CHECK(flags.numel() * 256 >= M, "gemm_ag: flags must hold one word per 256-row tile");
  const void* as[kMaxRanks] = {nullptr};
  uint32_t* pd[kMaxRanks] = {nullptr};
  for (int64_t i = 0; i < nr; ++i) {
    as[i] = (const void*)a_bufs[i];
    pd[i] = (uint32_t*)pads[i];
  }
  dtg::gemm_bf16_ag(as, b.data_ptr(), out.data_ptr(), M, N, K, b.stride(0), out.stride(0), b_kmajor, (int)nr, (int)rank,
                    (int)rows_per_peer, (uint32_t*)flags.data_ptr<int>(), (uint32_t)ag_epoch, pd, (uint32_t)bar_epoch,
                    (int)n_comm, stream(), bp);
}

// out = (residual +) the sum of parts [nparts, *out.shape], nparts in 1..8; every tensor bf16, contiguous and 16-byte
// aligned on out's device.  An empty out launches nothing.
void py_reduce_parts(const Tensor& parts, const c10::optional<Tensor>& residual, Tensor& out) {
  const Tensor* res = residual.has_value() ? &*residual : nullptr;
  check_dist("tp_reduce_parts", {}, 1, 0, &out,
             {{&parts, "parts", at::kBFloat16, true}, {&out, "out", at::kBFloat16, true},
              {res, "residual", at::kBFloat16, true}});
  TORCH_CHECK(parts.dim() == out.dim() + 1 && parts.size(0) >= 1 && parts.size(0) <= kMaxRanks &&
                  parts.sizes().slice(1) == out.sizes(),
              "tp_reduce_parts: parts must be [nparts, *out.shape] with 1..", kMaxRanks, " parts");
  TORCH_CHECK(!res || res->sizes() == out.sizes(), "tp_reduce_parts: residual must have out's shape");
  TORCH_CHECK(out.numel() % 8 == 0, "tp_reduce_parts: size must be a multiple of 8");
  if (out.numel() == 0) return;
  const c10::cuda::CUDAGuard guard(out.device());
  dtg::tp_reduce_parts(parts.data_ptr(), res ? res->data_ptr() : nullptr, out.data_ptr(), out.numel(),
                       (int)parts.size(0), stream());
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

// the per-row stats buffer of vocab_parallel CE: (max, sum-exp, target logit, mine) as float4 per row
void check_stats_ptr(uint64_t p, const char* who) {
  TORCH_CHECK(p != 0 && p % 16 == 0, who, ": every stats buffer must start at a 16-byte aligned address");
}

void py_vp_ce_stats(const Tensor& logits, const Tensor& targets, Tensor& stats, int64_t v0) {
  check_loss_args(logits, targets, "vp_ce_stats");
  const int64_t T = logits.size(0), Vl = logits.size(1);
  TORCH_CHECK(stats.is_cuda() && stats.device() == logits.device(), "vp_ce_stats: stats must be on logits' device");
  TORCH_CHECK(stats.scalar_type() == at::kFloat && stats.is_contiguous(), "vp_ce_stats: stats must be contiguous fp32");
  TORCH_CHECK(stats.numel() >= 4 * T, "vp_ce_stats: stats must hold 4 floats per row (", 4 * T, "), got ",
              stats.numel());
  check_stats_ptr((uint64_t)stats.data_ptr(), "vp_ce_stats");
  TORCH_CHECK(v0 >= 0 && v0 % Vl == 0, "vp_ce_stats: v0 must be a non-negative multiple of the shard width ", Vl,
              ", got ", v0);
  const c10::cuda::CUDAGuard guard(logits.device());
  dtg::vp_ce_stats(logits.data_ptr(), (const long long*)targets.data_ptr<int64_t>(), stats.data_ptr(), (int)T, (int)Vl,
                   (int)v0, stream());
}

Tensor py_vp_ce_grad(Tensor& logits, const Tensor& targets, const std::vector<uint64_t>& stats_ptrs, int64_t v0) {
  check_loss_args(logits, targets, "vp_ce_grad");
  const int64_t T = logits.size(0), Vl = logits.size(1), nr = (int64_t)stats_ptrs.size();
  TORCH_CHECK(nr == 1 || nr == 2 || nr == 4 || nr == 8, "vp_ce_grad: 1, 2, 4 or 8 ranks, got ", nr);
  for (uint64_t p : stats_ptrs) check_stats_ptr(p, "vp_ce_grad");
  TORCH_CHECK(v0 >= 0 && v0 % Vl == 0 && v0 / Vl < nr, "vp_ce_grad: v0 must be a multiple of the shard width ", Vl,
              " below ", nr, " shards, got ", v0);
  const c10::cuda::CUDAGuard guard(logits.device());
  if (T == 0) return torch::zeros({}, logits.options().dtype(at::kFloat));   // as with every target ignored
  Tensor scratch = torch::empty({T + 2}, logits.options().dtype(at::kFloat));
  float* sp = scratch.data_ptr<float>();
  const long long* tg = (const long long*)targets.data_ptr<int64_t>();
  dtg::ce_count_valid(tg, sp, (int)T, stream());
  dtg::vp_ce_grad(logits.data_ptr(), tg, plain(stats_ptrs), sp + 2, sp, (int)T, (int)Vl, (int)v0, (int)nr, stream());
  dtg::ce_finalize(sp + 2, sp, sp + 1, (int)T, stream());
  return scratch.slice(0, 1, 2).reshape({});
}

// the token layout of the hidden-parallel embedding: token t of the full batch lives in row t % rpp of rank t / rpp's
// [rpp, H] buffer, and this rank owns columns [rank * Hl, (rank + 1) * Hl)
void check_tp_tokens(int64_t T, const std::vector<uint64_t>& ptrs, int64_t rpp, int64_t H, int64_t Hl, int64_t rank,
                     const char* who) {
  const int64_t nr = (int64_t)ptrs.size();
  TORCH_CHECK(nr >= 1 && nr <= kMaxRanks, who, ": 1..", kMaxRanks, " ranks, got ", nr);
  for (uint64_t p : ptrs) TORCH_CHECK(p != 0 && p % 16 == 0, who, ": every rank's buffer must be 16-byte aligned");
  TORCH_CHECK(rank >= 0 && rank < nr, who, ": rank ", rank, " outside the ", nr, " ranks");
  TORCH_CHECK(rpp >= 1, who, ": rows per rank must be positive");
  TORCH_CHECK(T <= nr * rpp, who, ": ", T, " tokens do not fit ", nr, " ranks of ", rpp, " rows");
  TORCH_CHECK(H == nr * Hl, who, ": H (", H, ") must be the ranks times the shard width (", nr, " x ", Hl, ")");
}

void py_embed_fwd(const Tensor& ids, const Tensor& w, const std::vector<uint64_t>& dst_ptrs, int64_t rpp, int64_t H,
                  int64_t rank) {
  check_embedding_args(ids, w, "w", "tp_embed_fwd");
  check_tp_tokens(ids.numel(), dst_ptrs, rpp, H, w.size(1), rank, "tp_embed_fwd");
  const c10::cuda::CUDAGuard guard(w.device());
  dtg::tp_embed_fwd((const long long*)ids.data_ptr<int64_t>(), w.data_ptr(), plain(dst_ptrs), ids.numel(), w.size(0),
                    (int)rpp, (int)H, (int)w.size(1), (int)rank, stream());
}
// the staging rows and embedding_bwd's scratch live until the call returns (the caching allocator keeps them on this
// stream)
void py_embed_bwd(const Tensor& ids, const std::vector<uint64_t>& dx_ptrs, Tensor& dw, int64_t rpp, int64_t H,
                  int64_t rank, bool accumulate) {
  check_embedding_args(ids, dw, "dw", "tp_embed_bwd");
  const int64_t T = ids.numel(), V = dw.size(0), Hl = dw.size(1);
  check_tp_tokens(T, dx_ptrs, rpp, H, Hl, rank, "tp_embed_bwd");
  TORCH_CHECK(T < 0xFFFFFFFFLL, "tp_embed_bwd: too many tokens for 32-bit slots");
  const c10::cuda::CUDAGuard guard(dw.device());
  Tensor staging = torch::empty({T, Hl}, dw.options());
  Tensor slot = torch::empty({V}, dw.options().dtype(at::kInt));
  Tensor sums = torch::empty({T, Hl}, dw.options().dtype(at::kFloat));
  dtg::tp_embed_bwd((const long long*)ids.data_ptr<int64_t>(), plain(dx_ptrs), dw.data_ptr(), staging.data_ptr(),
                    reinterpret_cast<unsigned int*>(slot.data_ptr<int>()), sums.data_ptr<float>(), T, V, (int)rpp,
                    (int)H, (int)Hl, (int)rank, accumulate, stream());
}
}  // namespace

void bind_tp(pybind11::module_& m) {
  m.def("gemm_dist", &py_gemm_dist);
  m.def("gemm_ag", &py_gemm_ag, py::arg("a_bufs"), py::arg("b"), py::arg("out"), py::arg("b_kmajor"), py::arg("rank"),
        py::arg("rows_per_peer"), py::arg("flags"), py::arg("ag_epoch"), py::arg("pads"), py::arg("bar_epoch"),
        py::arg("n_comm"), py::arg("bias") = py::none());
  m.def("tp_reduce_parts", &py_reduce_parts);
  m.def("tp_reduce_mc", &py_reduce_mc);
  m.def("vp_ce_stats", &py_vp_ce_stats);
  m.def("vp_ce_grad", &py_vp_ce_grad);
  m.def("tp_embed_fwd", &py_embed_fwd);
  m.def("tp_embed_bwd", &py_embed_bwd, py::arg("ids"), py::arg("dx_ptrs"), py::arg("dw"), py::arg("rpp"), py::arg("H"),
        py::arg("rank"), py::arg("accumulate") = false);
}
}  // namespace dtg
