// Shared by the attention forward / backward kernels.
#pragma once
#include <cuda.h>

namespace dtg {
// TMA descriptor over a [B, S, heads, D] bf16 tensor (D = 64 or 128): dims {D, heads, S, B}, box {64, 1, rows, 1},
// 128-byte swizzle.  One [rows x D] head tile = D / 64 loads (columns 0-63, and 64-127 at D = 128).
CUtensorMap make_tmap_heads(const void* base, int B, int S, int heads, int box_rows, int D);
}  // namespace dtg
