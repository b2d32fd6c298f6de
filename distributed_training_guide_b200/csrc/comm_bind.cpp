// Symmetric-memory runtime (allocation outside the caching allocator, CUDA IPC export/import of
// peer mappings) and Python bindings of the NVLink collective kernels.
//
// Setup protocol (parallel/symm.py): every rank cudaMalloc's the same number of bytes, exports a
// 64-byte cudaIpcMemHandle, the handles are all-gathered through the torch.distributed store/NCCL
// bootstrap group, and each rank opens its peers' handles -> a table of N base pointers to the
// "same" buffer.  After that no library is involved: kernels address peers directly over NVLink.
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <pybind11/stl.h>
#include <torch/extension.h>

#include <cstring>
#include <mutex>
#include <unordered_map>

#include "comm.cuh"
#include "comm_api.h"
#include "common.cuh"

namespace dtg {
namespace {
using torch::Tensor;

std::mutex g_mu;
std::unordered_map<uint64_t, size_t> g_local;  // ptr -> bytes (owned allocations)
size_t g_local_bytes = 0;

inline cudaStream_t stream() { return at::cuda::getCurrentCUDAStream().stream(); }

// Allocate `nbytes` of device memory for peer mapping; returns (uint8 tensor view, ipc handle bytes).
std::tuple<Tensor, py::bytes> symm_alloc(int64_t nbytes, int64_t device) {
  const c10::cuda::CUDAGuard guard((c10::DeviceIndex)device);
  void* p = nullptr;
  const size_t bytes = ((size_t)nbytes + 511) & ~(size_t)511;
  DTG_CUDA_CHECK(cudaMalloc(&p, bytes));
  DTG_CUDA_CHECK(cudaMemset(p, 0, bytes));
  DTG_CUDA_CHECK(cudaDeviceSynchronize());
  cudaIpcMemHandle_t h;
  DTG_CUDA_CHECK(cudaIpcGetMemHandle(&h, p));
  {
    std::lock_guard<std::mutex> lk(g_mu);
    g_local[(uint64_t)p] = bytes;
    g_local_bytes += bytes;
  }
  auto deleter = [](void* q) {
    std::lock_guard<std::mutex> lk(g_mu);
    auto it = g_local.find((uint64_t)q);
    if (it != g_local.end()) {
      g_local_bytes -= it->second;
      g_local.erase(it);
    }
    cudaFree(q);
  };
  Tensor t = torch::from_blob(p, {(int64_t)bytes}, deleter,
                              torch::TensorOptions().dtype(torch::kUInt8).device(torch::kCUDA, (c10::DeviceIndex)device));
  return {t, py::bytes(reinterpret_cast<const char*>(&h), sizeof(h))};
}

// An independent tensor (own version counter, own autograd identity) over bytes [off, off + nbytes) of a chunk
// allocation; it keeps the chunk alive.  Sub-allocations must NOT be slices of one base tensor: an in-place write
// to a gradient buffer would then bump the version of every parameter saved for backward.
Tensor symm_alias(const Tensor& chunk, int64_t off, int64_t nbytes) {
  TORCH_CHECK(chunk.scalar_type() == at::kByte && off >= 0 && nbytes >= 0 && off + nbytes <= chunk.numel(), "bad alias");
  Tensor keep = chunk;
  return torch::from_blob((char*)chunk.data_ptr() + off, {nbytes}, [keep](void*) {}, chunk.options());
}

uint64_t symm_open(const std::string& handle, int64_t device) {
  TORCH_CHECK(handle.size() == sizeof(cudaIpcMemHandle_t), "bad IPC handle size");
  const c10::cuda::CUDAGuard guard((c10::DeviceIndex)device);
  cudaIpcMemHandle_t h;
  std::memcpy(&h, handle.data(), sizeof(h));
  void* p = nullptr;
  DTG_CUDA_CHECK(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
  return (uint64_t)p;
}

void symm_close(uint64_t ptr) { cudaIpcCloseMemHandle((void*)ptr); }

int64_t symm_allocated_bytes() { return (int64_t)g_local_bytes; }

SymmPtrs rotated(const std::vector<uint64_t>& ptrs, int rank) {
  SymmPtrs s{};
  const int n = (int)ptrs.size();
  TORCH_CHECK(n >= 1 && n <= kMaxRanks, "1..8 ranks supported");
  for (int k = 0; k < n; ++k) s.ptr[k] = (char*)ptrs[(rank + k) % n];
  return s;
}
SymmPads pads_of(const std::vector<uint64_t>& ptrs) {
  SymmPads s{};
  TORCH_CHECK(ptrs.size() <= (size_t)kMaxRanks, "1..8 ranks supported");
  for (size_t k = 0; k < ptrs.size(); ++k) s.ptr[k] = (uint32_t*)ptrs[k];
  return s;
}

// ---- argument checks of the peer-pointer collectives: each refuses before any launch ------------------------------
// The kernels index the peer and pad tables by rank (the barrier stores into every rank's pad), make 16-byte vector
// accesses at elem_off / shard_off and at every local operand, and take sizes and offsets as size_t, where a
// negative value would wrap into a huge one.

// 1..8 peers, rank in [0, nranks), one pad per peer; every entry a nonzero 16-byte aligned address
void check_peers(const char* who, const std::vector<uint64_t>& ptrs, const char* name,
                 const std::vector<uint64_t>& pads, int64_t rank) {
  const int64_t nr = (int64_t)ptrs.size();
  TORCH_CHECK(nr >= 1 && nr <= kMaxRanks, who, ": 1..", kMaxRanks, " ranks, got ", nr);
  TORCH_CHECK(rank >= 0 && rank < nr, who, ": rank ", rank, " outside the ", nr, " ranks");
  TORCH_CHECK((int64_t)pads.size() == nr, who, ": pads must have ", nr, " entries, got ", pads.size());
  for (uint64_t p : ptrs)
    TORCH_CHECK(p != 0 && p % 16 == 0, who, ": every entry of ", name, " must be a 16-byte aligned address");
  for (uint64_t p : pads)
    TORCH_CHECK(p != 0 && p % 16 == 0, who, ": every entry of pads must be a 16-byte aligned address");
}

// an element count (any value >= 0) or an element offset (a multiple of 8: one 16-byte vector)
void check_count(const char* who, const char* name, int64_t v) {
  TORCH_CHECK(v >= 0, who, ": ", name, " must not be negative, got ", v);
}
void check_offset(const char* who, const char* name, int64_t v) {
  TORCH_CHECK(v >= 0 && v % 8 == 0, who, ": ", name, " must be a non-negative multiple of 8, got ", v);
}

// a local operand: on the current device (where the kernel runs), contiguous, 16-byte aligned, of `dtype` unless
// that is Undefined
void check_local(const char* who, const char* name, const Tensor& t, at::ScalarType dtype = at::ScalarType::Undefined) {
  const c10::Device d(c10::kCUDA, c10::cuda::current_device());
  TORCH_CHECK(t.is_cuda() && t.device() == d, who, ": ", name, " must be on ", d);
  TORCH_CHECK(dtype == at::ScalarType::Undefined || t.scalar_type() == dtype, who, ": ", name, " must be ",
              c10::toString(dtype));
  TORCH_CHECK(t.is_contiguous(), who, ": ", name, " must be contiguous");
  TORCH_CHECK(reinterpret_cast<uintptr_t>(t.data_ptr()) % 16 == 0, who, ": ", name,
              " must start at a 16-byte aligned address");
}

// the barrier's timeout flag: an int32 word on the current device, or none
int* err_ptr(const char* who, const c10::optional<Tensor>& err) {
  if (!err.has_value()) return nullptr;
  const c10::Device d(c10::kCUDA, c10::cuda::current_device());
  TORCH_CHECK(err->is_cuda() && err->device() == d && err->scalar_type() == at::kInt && err->numel() >= 1, who,
              ": err must be an int32 tensor on ", d);
  return err->data_ptr<int>();
}

void allreduce_scale(const std::vector<uint64_t>& buf, const std::vector<uint64_t>& pads, int64_t elem_off, int64_t n,
                     double scale, int64_t rank, int64_t epoch, const c10::optional<Tensor>& err, int64_t blocks) {
  const char* who = "comm_allreduce_scale";
  check_peers(who, buf, "buf", pads, rank);
  check_offset(who, "elem_off", elem_off);
  check_count(who, "n", n);
  int* e = err_ptr(who, err);
  comm_allreduce_scale(rotated(buf, (int)rank), pads_of(pads), (size_t)elem_off, (size_t)n, (float)scale, (int)rank,
                       (int)buf.size(), (uint32_t)epoch, e, (int)blocks, stream());
}

void rs_adamw(const std::vector<uint64_t>& grads, const std::vector<uint64_t>& params,
              const c10::optional<Tensor>& param_local, Tensor& m, Tensor& v, bool push_params,
              const std::vector<uint64_t>& pads, int64_t elem_off, int64_t n, double lr, double b1, double b2, double eps,
              double wd, int64_t step, double grad_scale, int64_t rank, int64_t epoch,
              const c10::optional<Tensor>& err, int64_t blocks) {
  const char* who = "comm_rs_adamw";
  check_peers(who, grads, "grads", pads, rank);
  if (push_params) {
    TORCH_CHECK(params.size() == grads.size(), who, ": params must have ", grads.size(), " entries, got ",
                params.size());
    for (uint64_t p : params)
      TORCH_CHECK(p != 0 && p % 16 == 0, who, ": every entry of params must be a 16-byte aligned address");
  }
  check_offset(who, "elem_off", elem_off);
  check_count(who, "n", n);
  check_local(who, "m", m);
  check_local(who, "v", v);
  const bool fp32 = m.scalar_type() == at::kFloat;
  TORCH_CHECK(m.scalar_type() == v.scalar_type() && (fp32 || m.scalar_type() == at::kBFloat16), "bad state dtype");
  const int nr = (int)grads.size();
  TORCH_CHECK(m.numel() * nr == n && v.numel() * nr == n, "optimizer shard must hold n / nranks elements");
  AdamWHyper hp = make_adamw_hyper((float)lr, (float)b1, (float)b2, (float)eps, (float)wd, (int)step, (float)grad_scale);
  void* pl = nullptr;
  if (!push_params) {
    TORCH_CHECK(param_local.has_value() && param_local->numel() * nr == n, "param shard must hold n / nranks elements");
    check_local(who, "param_local", *param_local, at::kBFloat16);
    pl = param_local->data_ptr();
  }
  int* e = err_ptr(who, err);
  comm_rs_adamw(rotated(grads, (int)rank), push_params ? rotated(params, (int)rank) : SymmPtrs{}, pl, m.data_ptr(),
                v.data_ptr(), fp32, push_params, pads_of(pads), (size_t)elem_off, (size_t)n, hp, (int)rank, nr,
                (uint32_t)epoch, e, (int)blocks, stream());
}

// ---- NVLS (multicast) variants ----------------------------------------------------------------------------------
void nvls_allreduce_scale(uint64_t mc, const std::vector<uint64_t>& pads, int64_t elem_off, int64_t n, double scale,
                          int64_t rank, int64_t epoch, const c10::optional<Tensor>& err, int64_t blocks) {
  comm_nvls_allreduce_scale((void*)mc, pads_of(pads), (size_t)elem_off, (size_t)n, (float)scale, (int)rank,
                            (int)pads.size(), (uint32_t)epoch, err_ptr("comm_nvls_allreduce_scale", err), (int)blocks,
                            stream());
}

void nvls_rs_adamw(uint64_t grads_mc, uint64_t params_mc, uint64_t params_local, Tensor& m, Tensor& v, bool push_params,
                   const std::vector<uint64_t>& pads, int64_t elem_off, int64_t n, double lr, double b1, double b2,
                   double eps, double wd, int64_t step, double grad_scale, int64_t rank, int64_t epoch,
                   const c10::optional<Tensor>& err, int64_t blocks) {
  const bool fp32 = m.scalar_type() == at::kFloat;
  TORCH_CHECK(m.scalar_type() == v.scalar_type() && (fp32 || m.scalar_type() == at::kBFloat16), "bad state dtype");
  const int nr = (int)pads.size();
  TORCH_CHECK(m.numel() * nr == n && v.numel() * nr == n, "optimizer shard must hold n / nranks elements");
  AdamWHyper hp = make_adamw_hyper((float)lr, (float)b1, (float)b2, (float)eps, (float)wd, (int)step, (float)grad_scale);
  comm_nvls_rs_adamw((const void*)grads_mc, (void*)params_mc, (void*)params_local, m.data_ptr(), v.data_ptr(), fp32,
                     push_params, pads_of(pads), (size_t)elem_off, (size_t)n, hp, (int)rank, nr, (uint32_t)epoch,
                     err_ptr("comm_nvls_rs_adamw", err), (int)blocks, stream());
}

void allgather(const std::vector<uint64_t>& shards, Tensor& full, const std::vector<uint64_t>& pads, int64_t shard_off,
               int64_t per, int64_t rank, int64_t epoch, const c10::optional<Tensor>& err, bool barrier,
               int64_t blocks) {
  const char* who = "comm_allgather";
  check_peers(who, shards, "shards", pads, rank);
  check_offset(who, "shard_off", shard_off);
  check_count(who, "per", per);
  check_local(who, "full", full, at::kBFloat16);
  TORCH_CHECK(full.numel() >= per * (int64_t)shards.size(), "full buffer too small");
  int* e = err_ptr(who, err);
  if (blocks <= 0) {  // copy-engine variant
    comm_allgather_ce(rotated(shards, (int)rank), full.data_ptr(), pads_of(pads), (size_t)shard_off, (size_t)per,
                      (int)rank, (int)shards.size(), (uint32_t)epoch, e, barrier, stream());
    return;
  }
  comm_allgather(rotated(shards, (int)rank), full.data_ptr(), pads_of(pads), (size_t)shard_off, (size_t)per, (int)rank,
                 (int)shards.size(), (uint32_t)epoch, e, barrier, (int)blocks, stream());
}

void reduce_scatter(const std::vector<uint64_t>& grads, Tensor& out, const std::vector<uint64_t>& pads, int64_t elem_off,
                    int64_t n, double scale, int64_t rank, int64_t epoch, const c10::optional<Tensor>& err,
                    int64_t blocks) {
  const char* who = "comm_reduce_scatter";
  check_peers(who, grads, "grads", pads, rank);
  check_offset(who, "elem_off", elem_off);
  check_count(who, "n", n);
  check_local(who, "out", out, at::kBFloat16);
  TORCH_CHECK(out.numel() * (int64_t)grads.size() == n, "out must be a contiguous bf16 shard of n / nranks elements");
  int* e = err_ptr(who, err);
  comm_reduce_scatter(rotated(grads, (int)rank), out.data_ptr(), pads_of(pads), (size_t)elem_off, (size_t)n,
                      (float)scale, (int)rank, (int)grads.size(), (uint32_t)epoch, e, (int)blocks, stream());
}

void barrier(const std::vector<uint64_t>& pads, int64_t rank, int64_t epoch, const c10::optional<Tensor>& err) {
  check_peers("comm_barrier", pads, "pads", pads, rank);
  comm_barrier(pads_of(pads), (int)rank, (int)pads.size(), (uint32_t)epoch, err_ptr("comm_barrier", err), stream());
}

// ---- gradient clipping (grad_clip.cu) ---------------------------------------------------------------------------
void check_clip_tables(const Tensor& ranges, const Tensor& partials, int64_t blocks) {
  TORCH_CHECK(ranges.is_cuda() && ranges.scalar_type() == at::kLong && ranges.is_contiguous() && ranges.dim() == 2 &&
                  ranges.size(1) == 2,
              "ranges must be a contiguous int64 [R, 2] CUDA tensor");
  TORCH_CHECK(partials.is_cuda() && partials.scalar_type() == at::kDouble && partials.is_contiguous() &&
                  partials.numel() >= blocks,
              "partials must be a contiguous fp64 CUDA tensor of at least `blocks` elements");
}

void reduce_sumsq(const std::vector<uint64_t>& buf, const std::vector<uint64_t>& pads, int64_t elem_off, int64_t n,
                  double scale, bool broadcast, const Tensor& ranges, Tensor& partials, int64_t rank, int64_t epoch,
                  const c10::optional<Tensor>& err, int64_t blocks) {
  const char* who = "comm_reduce_sumsq";
  check_peers(who, buf, "buf", pads, rank);
  check_offset(who, "elem_off", elem_off);
  check_count(who, "n", n);
  check_clip_tables(ranges, partials, blocks);
  int* e = err_ptr(who, err);
  comm_reduce_sumsq(rotated(buf, (int)rank), pads_of(pads), (size_t)elem_off, (size_t)n, (float)scale, broadcast,
                    (const long long*)ranges.data_ptr<int64_t>(), (int)ranges.size(0), partials.data_ptr<double>(), (int)rank,
                    (int)buf.size(), (uint32_t)epoch, e, (int)blocks, stream());
}

void nvls_reduce_sumsq(uint64_t mc, uint64_t local, const std::vector<uint64_t>& pads, int64_t elem_off, int64_t n,
                       double scale, bool broadcast, const Tensor& ranges, Tensor& partials, int64_t rank,
                       int64_t epoch, const c10::optional<Tensor>& err, int64_t blocks) {
  check_clip_tables(ranges, partials, blocks);
  comm_nvls_reduce_sumsq((void*)mc, (void*)local, pads_of(pads), (size_t)elem_off, (size_t)n, (float)scale, broadcast,
                         (const long long*)ranges.data_ptr<int64_t>(), (int)ranges.size(0), partials.data_ptr<double>(), (int)rank,
                         (int)pads.size(), (uint32_t)epoch, err_ptr("comm_nvls_reduce_sumsq", err), (int)blocks, stream());
}

// slots: every rank's slot buffer in RANK order (not rotated)
void clip_finalize(const Tensor& partials, const std::vector<uint64_t>& slots, const std::vector<uint64_t>& pads,
                   int64_t parity, double norm_scale, double max_norm, Tensor& out, int64_t rank, int64_t epoch,
                   const c10::optional<Tensor>& err) {
  TORCH_CHECK(partials.is_cuda() && partials.scalar_type() == at::kDouble && partials.is_contiguous(),
              "partials must be a contiguous fp64 CUDA tensor");
  TORCH_CHECK(out.is_cuda() && out.scalar_type() == at::kFloat && out.is_contiguous() && out.numel() >= 2,
              "out must be a contiguous fp32 CUDA tensor of 2 elements (norm, coef)");
  TORCH_CHECK(slots.size() == pads.size() && slots.size() >= 1 && slots.size() <= (size_t)kMaxRanks,
              "one slot buffer per rank");
  check_peers("comm_clip_finalize", slots, "slots", pads, rank);
  int* e = err_ptr("comm_clip_finalize", err);
  SymmPtrs sp{};
  for (size_t k = 0; k < slots.size(); ++k) sp.ptr[k] = (char*)slots[k];
  comm_clip_finalize(partials.data_ptr<double>(), (int)partials.numel(), sp, pads_of(pads), (int)parity,
                     (float)norm_scale, (float)max_norm, out.data_ptr<float>(), (int)rank, (int)pads.size(),
                     (uint32_t)epoch, e, stream());
}

// AdamW on p_src / g / m / v (one rank's range) with g *= coef[0]; the new parameters go to every address of `dst`
// (the same range on each replica), or through the multicast address `dst_mc` when it is not 0.
void adamw_clip_(const std::vector<uint64_t>& dst, uint64_t dst_mc, const Tensor& p_src, const Tensor& g, Tensor& m,
                 Tensor& v, double lr, double b1, double b2, double eps, double wd, int64_t step, double grad_scale,
                 const Tensor& coef) {
  for (const Tensor* t : {&p_src, &g}) {
    TORCH_CHECK(t->is_cuda() && t->scalar_type() == at::kBFloat16 && t->is_contiguous() &&
                    (reinterpret_cast<uintptr_t>(t->data_ptr()) & 15) == 0,
                "adamw_clip: parameters and gradients must be contiguous, 16-byte aligned bf16 CUDA tensors");
  }
  const bool fp32 = m.scalar_type() == at::kFloat;
  TORCH_CHECK(m.scalar_type() == v.scalar_type() && (fp32 || m.scalar_type() == at::kBFloat16), "bad state dtype");
  check_local("comm_adamw_clip", "m", m);
  check_local("comm_adamw_clip", "v", v);
  TORCH_CHECK(p_src.numel() == g.numel() && g.numel() == m.numel() && m.numel() == v.numel(), "size mismatch");
  TORCH_CHECK(coef.is_cuda() && coef.scalar_type() == at::kFloat && coef.numel() >= 1, "coef must be fp32 on the device");
  TORCH_CHECK(dst_mc != 0 || (dst.size() >= 1 && dst.size() <= (size_t)kMaxRanks), "1..8 destinations");
  for (uint64_t p : dst)
    TORCH_CHECK(p != 0 && p % 16 == 0, "comm_adamw_clip: every entry of dst must be a 16-byte aligned address");
  SymmPtrs sp{};
  for (size_t k = 0; k < dst.size() && k < (size_t)kMaxRanks; ++k) sp.ptr[k] = (char*)dst[k];
  AdamWHyper hp = make_adamw_hyper((float)lr, (float)b1, (float)b2, (float)eps, (float)wd, (int)step, (float)grad_scale);
  adamw_clip(sp, (void*)dst_mc, p_src.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), fp32, p_src.numel(), hp,
             coef.data_ptr<float>(), (int)dst.size(), stream());
}

}  // namespace

void bind_comm(pybind11::module_& m) {
  m.def("symm_alloc", &symm_alloc);
  m.def("symm_open", &symm_open);
  m.def("symm_alias", &symm_alias);
  m.def("symm_close", &symm_close);
  m.def("symm_allocated_bytes", &symm_allocated_bytes);
  m.attr("SYMM_PAD_BYTES") = (int64_t)kPadBytes;
  m.attr("SYMM_MAX_CHANNELS") = (int64_t)kMaxChannels;
  m.def("comm_allreduce_scale", &allreduce_scale);
  m.def("comm_rs_adamw", &rs_adamw);
  m.def("comm_allgather", &allgather);
  m.def("comm_nvls_allreduce_scale", &nvls_allreduce_scale);
  m.def("comm_nvls_rs_adamw", &nvls_rs_adamw);
  m.def("comm_reduce_scatter", &reduce_scatter);
  m.def("comm_barrier", &barrier);
  m.def("comm_reduce_sumsq", &reduce_sumsq);
  m.def("comm_nvls_reduce_sumsq", &nvls_reduce_sumsq);
  m.def("comm_clip_finalize", &clip_finalize);
  m.def("comm_adamw_clip", &adamw_clip_);
}
}  // namespace dtg
