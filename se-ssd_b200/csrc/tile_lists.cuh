// tile_lists.cuh -- the tile-list record (sessd_rulebook_tile_lists, rulebook.cu): the neighbour table regrouped by tile of kTlRows output
// rows, read by the pair-proportional tensor-core conv (spconv_cg.cu) and the weight gradient (spconv_grad.cu).  One record per tile, in
// 32-bit words:
//   [0, 32)                         pair count per kernel offset (kvol <= 27 < 32)
//   [kTlMask, kTlMask + 4 kvol)     128-bit row mask per offset: tile rows that have a neighbour at offset k
//   [kTlHeader, kTlHeader + pairs)  the pairs of offset 0, then of offset 1, ..., each tl_entry(input row, tile row), ascending tile row
// tests/cases.py restates the format independently.
#pragma once
#include "common.cuh"

namespace sessd {

constexpr int kTlRows = 128;                 // output rows per record
constexpr int kTlMask = 32;                  // first word of the row masks
constexpr int kTlHeader = kTlMask + 4 * 32;  // first word of the pair entries
static_assert(kTlRows == 1 << 7, "an entry keeps the tile row in its low 7 bits");
__host__ __device__ constexpr int tile_list_stride(int kvol) { return kTlHeader + kTlRows * kvol; }

__device__ __forceinline__ unsigned int tl_entry(int in_row, int tile_row) { return ((unsigned int)in_row << 7) | (unsigned int)tile_row; }
__device__ __forceinline__ unsigned int tl_in_row(unsigned int e) { return e >> 7; }
__device__ __forceinline__ unsigned int tl_tile_row(unsigned int e) { return e & (kTlRows - 1u); }

// first entry of offset k in a record's pair list: after the pairs of the offsets < k
__device__ __forceinline__ int tl_offset_start(const unsigned int *rec, int k) {
    int s = 0;
    for (int j = 0; j < k; ++j) s += (int)__ldg(rec + j);
    return s;
}

}  // namespace sessd
