// Tensor maps (TMA descriptors) of the attention kernels: 128-byte-swizzled boxes (CU_TENSOR_MAP_SWIZZLE_128B).
// A box row is one whole 128-byte line (64 16-bit elements).
// Shared-memory layout of a box: row r at r * 128, its 16-byte chunk c at ((c ^ (r & 7)) * 16) - the canonical wgmma
// SWIZZLE_128B layout (K-major operands, and MN-major operands whose MN extent is 64; wgmma.cuh make_desc_sw128).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace ub {

// [B, L, H, D] tensor (D % 8 == 0, heads contiguous), box = box_rows x 64 columns of one (batch, head); coordinates
// {col0 (0 or 64), head, row0, batch}.  Columns at or past D read as zeros.
bool make_head_tile_map_sw128(CUtensorMap* map, const void* base, bool bf16, int B, int L, int H, int D, long long sb,
                              long long sl, long long sh, int box_rows);
// bias [NB, Lq, Lk]: box = 64 rows x 64 columns (a 64 x 128 tile is two boxes); coordinates {key0, q0, nb}.
bool make_bias_tile_map_sw128(CUtensorMap* map, const void* base, bool bf16, int NB, int Lq, int Lk);

}  // namespace ub
