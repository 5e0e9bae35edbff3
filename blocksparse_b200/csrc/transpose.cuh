// transpose_0213 / transpose_2d (bst_transpose_0213 in include/bsmm_b200.h): y = x viewed as (D0, D1, D2, D3) with dims 1
// and 2 swapped, y (D0, D2, D1, D3). A pure copy: the kernels move bits and never convert, so one kernel serves every dtype
// of the same width. Two routes, picked from the row of D3 elements (a "cell"):
//   * rows (cells of >= TR_ROW_BYTES): every output cell is a contiguous copy of one input cell, in words of the widest
//     of 16 / 8 / 4 / 2 bytes that the cell size and both base pointers allow; cells of fewer than TR_THREADS words share
//     a CTA, so a warp writes several consecutive output cells, one contiguous run;
//   * tile (narrower cells, D3 = 1 being transpose_2d): a TR_TILE x TR_TILE tile of cells of one (D1, D2) slice is read
//     row by row into shared memory and written column by column, so both sides are contiguous runs of TR_TILE cells.
//     Shared memory holds one 32-bit word per element with a row pitch of (TR_TILE + 1) * D3 words: the column reads
//     of a warp hit 32 consecutive words modulo 32 banks, so neither phase has bank conflicts.
#pragma once
#include <algorithm>
#include "common.cuh"

namespace bsmm {

constexpr int TR_ROW_BYTES = 16;
constexpr int TR_THREADS = 256;
constexpr int TR_TILE = 32;
constexpr long long TR_MAX_GRID = 1 << 20;    // CTAs of a launch; both kernels loop over the rest

// rpb output cells per CTA (a power of two), TR_THREADS / rpb threads per cell. I: the index type, 32-bit whenever the
// cell count allows, so that the per-cell divisions are cheap.
template <typename W, typename I>
__global__ void __launch_bounds__(TR_THREADS) transpose_rows_kernel(const W* __restrict__ x, W* __restrict__ y, I D1, I D2,
                                                                    I cells, long long wpc, int rpb) {
  const int lanes = TR_THREADS / rpb;
  const int r = threadIdx.x / lanes, l = threadIdx.x % lanes;
  for (I oc = (I)blockIdx.x * rpb + r; oc < cells; oc += (I)gridDim.x * rpb) {
    const I d1 = oc % D1, t = oc / D1, d2 = t % D2, d0 = t / D2;
    const W* src = x + ((long long)((d0 * D1 + d1) * D2 + d2)) * wpc;
    W* dst = y + (long long)oc * wpc;
    for (long long w = l; w < wpc; w += lanes) __stcs(dst + w, __ldcs(src + w));
  }
}

// E: the element's bits (uint16_t or uint32_t); the tile covers cells (d1, d2) in [d1t, d1t + 32) x [d2t, d2t + 32).
template <typename E, int D3>
__global__ void __launch_bounds__(TR_THREADS) transpose_tile_kernel(const E* __restrict__ x, E* __restrict__ y, long long D1,
                                                                    long long D2, long long tiles1, long long tiles2,
                                                                    long long tiles) {
  constexpr int RUN = TR_TILE * D3;                // elements of a tile row: TR_TILE cells
  constexpr int PITCH = (TR_TILE + 1) * D3;
  __shared__ uint32_t sh[TR_TILE * PITCH];
  for (long long tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
    const long long t2 = tile % tiles2, rest = tile / tiles2, t1 = rest % tiles1, d0 = rest / tiles1;
    const long long d1t = t1 * TR_TILE, d2t = t2 * TR_TILE;
    const int n1 = (int)(D1 - d1t < TR_TILE ? D1 - d1t : TR_TILE), n2 = (int)(D2 - d2t < TR_TILE ? D2 - d2t : TR_TILE);
    const E* src = x + ((d0 * D1 + d1t) * D2 + d2t) * D3;            // row r of the tile: src + r * D2 * D3
    for (int i = threadIdx.x; i < TR_TILE * RUN; i += TR_THREADS) {
      const int r = i / RUN, e = i % RUN;
      if (r < n1 && e < n2 * D3) sh[r * PITCH + e] = __ldcs(src + r * D2 * D3 + e);
    }
    __syncthreads();
    E* dst = y + ((d0 * D2 + d2t) * D1 + d1t) * D3;                  // row c of the output tile: dst + c * D1 * D3
    for (int i = threadIdx.x; i < TR_TILE * RUN; i += TR_THREADS) {
      const int c = i / RUN, e = i % RUN, r = e / D3, s = e % D3;
      if (c < n2 && e < n1 * D3) __stcs(dst + c * D1 * D3 + e, (E)sh[r * PITCH + c * D3 + s]);
    }
    __syncthreads();
  }
}

template <typename W>
int launch_transpose_rows(const void* x, void* y, long long D1, long long D2, long long cells, long long wpc, cudaStream_t s) {
  int rpb = 1;
  while (rpb < TR_THREADS && (long long)(TR_THREADS / rpb / 2) >= wpc) rpb <<= 1;
  const unsigned grid = (unsigned)std::min((cells + rpb - 1) / rpb, TR_MAX_GRID);
  if (cells < 0x7fffffffLL)                    // oc + the grid stride stays below 2^32
    transpose_rows_kernel<W, unsigned><<<grid, TR_THREADS, 0, s>>>((const W*)x, (W*)y, (unsigned)D1, (unsigned)D2,
                                                                   (unsigned)cells, wpc, rpb);
  else
    transpose_rows_kernel<W, unsigned long long><<<grid, TR_THREADS, 0, s>>>((const W*)x, (W*)y, D1, D2, cells, wpc, rpb);
  return check_launch("transpose_rows");
}

template <typename E, int D3>
int launch_transpose_tile_d3(const void* x, void* y, long long D0, long long D1, long long D2, cudaStream_t s) {
  const long long tiles1 = (D1 + TR_TILE - 1) / TR_TILE, tiles2 = (D2 + TR_TILE - 1) / TR_TILE, tiles = D0 * tiles1 * tiles2;
  const unsigned grid = (unsigned)std::min(tiles, TR_MAX_GRID);
  transpose_tile_kernel<E, D3><<<grid, TR_THREADS, 0, s>>>((const E*)x, (E*)y, D1, D2, tiles1, tiles2, tiles);
  return check_launch("transpose_tile");
}

// D3 * sizeof(E) < TR_ROW_BYTES: D3 in 1..7 for 2-byte elements, 1..3 for 4-byte ones
template <typename E>
int launch_transpose_tile(const void* x, void* y, long long D0, long long D1, long long D2, int D3, cudaStream_t s) {
  switch (D3) {
    case 1: return launch_transpose_tile_d3<E, 1>(x, y, D0, D1, D2, s);
    case 2: return launch_transpose_tile_d3<E, 2>(x, y, D0, D1, D2, s);
    case 3: return launch_transpose_tile_d3<E, 3>(x, y, D0, D1, D2, s);
  }
  if constexpr (sizeof(E) == 2) {
    switch (D3) {
      case 4: return launch_transpose_tile_d3<E, 4>(x, y, D0, D1, D2, s);
      case 5: return launch_transpose_tile_d3<E, 5>(x, y, D0, D1, D2, s);
      case 6: return launch_transpose_tile_d3<E, 6>(x, y, D0, D1, D2, s);
      case 7: return launch_transpose_tile_d3<E, 7>(x, y, D0, D1, D2, s);
    }
  }
  return fail(BSMM_E_ARG, "transpose_tile: no kernel for D3 = %d of %d-byte elements", D3, (int)sizeof(E));
}

// Picks the route and the word width. esize: bytes per element (2 or 4).
inline int launch_transpose_0213(int esize, const void* x, void* y, long long D0, long long D1, long long D2, long long D3,
                                 cudaStream_t s) {
  const long long cell = D3 * esize;
  if (cell < TR_ROW_BYTES) {
    if (esize == 2) return launch_transpose_tile<uint16_t>(x, y, D0, D1, D2, (int)D3, s);
    return launch_transpose_tile<uint32_t>(x, y, D0, D1, D2, (int)D3, s);
  }
  const uintptr_t bits = (uintptr_t)x | (uintptr_t)y | (uintptr_t)cell;
  const long long cells = D0 * D1 * D2;
  if (!(bits & 15)) return launch_transpose_rows<uint4>(x, y, D1, D2, cells, cell / 16, s);
  if (!(bits & 7))  return launch_transpose_rows<uint2>(x, y, D1, D2, cells, cell / 8, s);
  if (!(bits & 3))  return launch_transpose_rows<uint32_t>(x, y, D1, D2, cells, cell / 4, s);
  return launch_transpose_rows<uint16_t>(x, y, D1, D2, cells, cell / 2, s);
}

}  // namespace bsmm
