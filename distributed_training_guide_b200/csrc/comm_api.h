// NVLink symmetric-memory runtime + collective kernels: Python binding entry point.
#pragma once
#include <pybind11/pybind11.h>

namespace at {
class Tensor;
}

namespace dtg {
// Argument checks shared by the plain and tensor-parallel bindings (bind.cpp); each refuses before any launch.
// logits: bf16 [T, V] contiguous, 16-byte aligned, V a positive multiple of 8; targets: int64 [T] contiguous on
// logits' device.
void check_loss_args(const at::Tensor& logits, const at::Tensor& targets, const char* who);
// ids: int64 contiguous on the table's device; table (w or dw): bf16 [V, H] contiguous, 16-byte aligned, H % 8 == 0.
void check_embedding_args(const at::Tensor& ids, const at::Tensor& table, const char* table_name, const char* who);
void bind_comm(pybind11::module_& m);
void bind_attention(pybind11::module_& m);
void bind_tp(pybind11::module_& m);
void bind_dataloader(pybind11::module_& m);
void bind_symm_vmm(pybind11::module_& m);
void bind_moe(pybind11::module_& m);
}  // namespace dtg
