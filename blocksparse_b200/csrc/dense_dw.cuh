// Dense weight-gradient GEMM U[C][K] = sum_n X[n][c] * E[n][k] in fp32, split over the minibatch (dw_matmul_large_n).
//   Replaces Gemm_TN (reference src/matmul_op_gpu.cu:309-364: hmma_gemm_64x64x32_TN_vec8 and gemm_32x32x32_TN_vec4),
//   launched by DwMatmulLargeNOp (src/matmul_op.cc).
//
// Minibatch split (dense_dw_split): the N rows are cut into S segments of whole 64-row stages, and every (output tile,
// segment) pair is one work item.  S depends on (N, C, K, route) only -- never on the SM count or BSMM_SM_MARGIN -- so
// U is bitwise the same on every H100, under any margin, on any stream and in a replayed graph.  Only the grid (the
// number of persistent CTAs walking the items) follows the SM count.
//   S == 1: each item writes its tile of U.
//   S  > 1: item (tile, s) writes its fp32 partial into slice s of the workspace ([S][C][K]); dense_dw_reduce_kernel
//           then adds the S slices in segment order.  No float atomics, and no CTA ever waits on another.
// Routes:
//   wgmma_dense_dw  fp16 / bf16 with C % 8 == 0, K % 8 == 0, 16-byte aligned operands and N < 2^31 (the TMA row-pitch,
//                   address and coordinate rules).  Tiles of 128 C-rows x up to 256 K-columns on the producer /
//                   consumer ring of tc_updat.cuh: TMA boxes of 64 features x 64 rows with 128-byte swizzle, both
//                   operands MN-major; each consumer warpgroup owns 64 rows and runs one wgmma per K = 16 step, as wide
//                   (64 / 128 / 192 / 256) as the tile's columns need.  Rows and columns past the edges are TMA's zero
//                   fill; stores are masked.
//   fma_dense_dw    everything else (fp32, which the reference also runs on CUDA cores, and 16-bit shapes TMA cannot
//                   take): 64 x 64 tiles, true fp32 FMA in row order, 64-bit offsets.
#pragma once
#include <climits>
#include "tc.cuh"

namespace bsmm {

constexpr long long DW_TARGET_ITEMS = 264;       // two waves of the H100 SXM's 132 SMs
constexpr long long DW_MIN_SEG_ROWS = 1024;      // 16 stages: keeps the ring's fill and the partial writes amortised
constexpr long long DW_STAGE_ROWS = 64;
constexpr int DW_TC_TM = 128, DW_TC_TN = 256, DW_FMA_TM = 64, DW_FMA_TN = 64;

struct DwSplit {
  long long tiles_k, tiles;   // output tiles along K, in all
  long long stages;           // 64-row stages of the minibatch
  long long seg_stages, S;    // stages per segment (the last may be shorter), segments
};

// S = max(1, min(TARGET / tiles, N / MIN_SEG)), then evened out over whole stages so that no segment is empty.
// S > 1 only when tiles < TARGET, so tiles * S <= TARGET and the workspace S * C * K * 4 <= TARGET * TM * TN * 4 bytes.
inline DwSplit dense_dw_split(long long N, long long C, long long K, bool tc) {
  const long long tm = tc ? DW_TC_TM : DW_FMA_TM, tn = tc ? DW_TC_TN : DW_FMA_TN;
  DwSplit d;
  d.tiles_k = (K + tn - 1) / tn;
  d.tiles = (C + tm - 1) / tm * d.tiles_k;
  d.stages = (N + DW_STAGE_ROWS - 1) / DW_STAGE_ROWS;
  long long s0 = d.tiles > 0 ? DW_TARGET_ITEMS / d.tiles : 1;
  if (N / DW_MIN_SEG_ROWS < s0) s0 = N / DW_MIN_SEG_ROWS;
  if (s0 < 1) s0 = 1;
  d.seg_stages = (d.stages + s0 - 1) / s0;
  d.S = d.seg_stages > 0 ? (d.stages + d.seg_stages - 1) / d.seg_stages : 1;
  return d;
}
inline size_t dense_dw_workspace(long long N, long long C, long long K, bool tc) {
  const DwSplit d = dense_dw_split(N, C, K, tc);
  return d.S > 1 ? (size_t)d.S * (size_t)C * (size_t)K * sizeof(float) : 0;
}
// The shape rules of the wgmma route (the pointer rules are checked at the call).
inline bool dense_dw_tc_shape(int dtype, long long N, int C, int K) {
  return dtype != BSMM_F32 && C % 8 == 0 && K % 8 == 0 && N <= INT_MAX;
}

struct DenseDwParams {
  float* out;                 // U when S == 1, else the workspace
  long long C, K, N;
  long long stages, seg_stages;
  int tiles, tiles_k, n_items;  // items segment-major: item i = (tile i % tiles, segment i / tiles)
};

// ---- wgmma route ------------------------------------------------------------------------------------------------
constexpr int DW_THREADS = 3 * 128;   // one producer warpgroup, two consumer warpgroups
constexpr int DW_STAGES = 4;
constexpr int DW_PRODUCER_REGS = 40, DW_CONSUMER_REGS = 232;
struct DwShape {
  static constexpr uint32_t BOX = 64 * 64 * 2;      // 64 features x 64 rows, 128-byte rows
  static constexpr uint32_t ABYTES = 2 * BOX;       // 128 C-rows
  static constexpr uint32_t STAGE = ABYTES + 4 * BOX;
  static constexpr size_t SMEM = DW_STAGES * STAGE + SMEM_ALIGN_SLACK;
};
struct DenseDwTmaps { CUtensorMap x, e; };

struct DwItem { long long c0, k0, first; int n_st, nch; };
__device__ __forceinline__ DwItem dense_dw_item(const DenseDwParams& p, int i, int tm, int tn) {
  const int tile = i % p.tiles, seg = i / p.tiles;
  DwItem it;
  it.c0 = (long long)(tile / p.tiles_k) * tm;
  it.k0 = (long long)(tile % p.tiles_k) * tn;
  it.first = (long long)seg * p.seg_stages;
  const long long left = p.stages - it.first;
  it.n_st = (int)(left < p.seg_stages ? left : p.seg_stages);
  const long long cols = p.K - it.k0 < tn ? p.K - it.k0 : tn;
  it.nch = (int)((cols + 63) / 64);
  return it;
}

// One item of one consumer warpgroup: rows 64cw..64cw+63 of the tile x NCH*64 columns, reduced over the n_st stages at
// ring positions g0, g0 + 1, ...; then its masked part of the store.
template <int NCH, bool BF16>
__device__ __forceinline__ void dense_dw_tile(const DenseDwParams& p, float* out, long long c0, long long k0, uint32_t base,
                                              uint64_t* full, uint64_t* empty, uint32_t g0, int n_st, int cw, int warp, int lane) {
  constexpr int ST = DW_STAGES;
  float acc[NCH * 32];
#pragma unroll
  for (int i = 0; i < NCH * 32; ++i) acc[i] = 0.f;

  for (int ch = 0; ch < n_st; ++ch) {
    const uint32_t g = g0 + ch;
    const uint32_t st = base + (g % ST) * DwShape::STAGE;
    if (!ptx::mbar_wait(&full[g % ST], (g / ST) & 1)) g_tc_error = 61;
    ptx::wg_fence();
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
      const uint64_t adesc = ptx::make_desc(st + cw * DwShape::BOX + ks * 2048, DwShape::BOX, 1024, ptx::SWZ_128B);
      const uint64_t bdesc = ptx::make_desc(st + DwShape::ABYTES + ks * 2048, DwShape::BOX, 1024, ptx::SWZ_128B);
      ptx::wgmma<BF16, 1, 1, NCH * 64>(acc, adesc, bdesc);
    }
    ptx::wg_commit();
    ptx::wg_wait<1>();                                // the MMAs of the previous stage have retired: hand it back
    if (ch > 0 && lane == 0) ptx::mbar_arrive(&empty[(g - 1) % ST]);
  }
  ptx::wg_wait<0>();
  if (lane == 0) ptx::mbar_arrive(&empty[(g0 + n_st - 1) % ST]);
  ptx::wg_fence_regs(acc);

  // acc[4j + 2h + e] = D[16 warp + lane/4 + 8h][8j + 2(lane % 4) + e]; K % 8 == 0, so col < K covers col + 1 too
  const long long r0 = c0 + cw * 64 + warp * 16 + lane / 4;
#pragma unroll
  for (int j = 0; j < NCH * 8; ++j) {
    const long long col = k0 + 8 * j + 2 * (lane % 4);
    if (col >= p.K) continue;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const long long r = r0 + 8 * h;
      if (r < p.C) *reinterpret_cast<float2*>(out + r * p.K + col) = make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
    }
  }
}

template <bool BF16>
__global__ void __launch_bounds__(DW_THREADS, 1)
wgmma_dense_dw_kernel(const __grid_constant__ DenseDwParams p, const __grid_constant__ DenseDwTmaps maps) {
  constexpr int ST = DW_STAGES;
  extern __shared__ uint8_t smem_raw[];
  __shared__ uint64_t full[ST], empty[ST];
  const uint32_t base = aligned_smem_base(smem_raw);
  const int tid = threadIdx.x, wg = tid / 128;

  if (tid == 0) {
    for (int i = 0; i < ST; ++i) {
      ptx::mbar_init(&full[i], 1);
      ptx::mbar_init(&empty[i], 8);                   // one arrival per consumer warp
    }
    ptx::fence_mbar_init();
  }
  __syncthreads();

  if (wg == 0) {
    ptx::setmaxnreg_dec<DW_PRODUCER_REGS>();
    if (tid != 0) return;
    uint32_t g = 0;                                   // ring position, continued across the CTA's items
    for (int i = blockIdx.x; i < p.n_items; i += gridDim.x) {
      const DwItem it = dense_dw_item(p, i, DW_TC_TM, DW_TC_TN);
      const uint32_t tx = DwShape::ABYTES + (uint32_t)it.nch * DwShape::BOX;
      for (int s = 0; s < it.n_st; ++s, ++g) {
        const uint32_t slot = g % ST;
        if (g >= ST && !ptx::mbar_wait(&empty[slot], (g / ST - 1) & 1)) g_tc_error = 62;
        const uint32_t st = base + slot * DwShape::STAGE;
        uint64_t* bar = &full[slot];
        const int n0 = (int)((it.first + s) * DW_STAGE_ROWS);
        ptx::mbar_expect_tx(bar, tx);
        ptx::tma_load_2d(st, &maps.x, bar, (int)it.c0, n0);
        ptx::tma_load_2d(st + DwShape::BOX, &maps.x, bar, (int)it.c0 + 64, n0);
        for (int j = 0; j < it.nch; ++j)
          ptx::tma_load_2d(st + DwShape::ABYTES + j * DwShape::BOX, &maps.e, bar, (int)it.k0 + 64 * j, n0);
      }
    }
    return;
  }

  ptx::setmaxnreg_inc<DW_CONSUMER_REGS>();
  const int cw = wg - 1, warp = (tid / 32) % 4, lane = tid % 32;
  uint32_t g = 0;
  for (int i = blockIdx.x; i < p.n_items; i += gridDim.x) {
    const DwItem it = dense_dw_item(p, i, DW_TC_TM, DW_TC_TN);
    float* out = p.out + (long long)(i / p.tiles) * p.C * p.K;
    switch (it.nch) {
      case 1:  dense_dw_tile<1, BF16>(p, out, it.c0, it.k0, base, full, empty, g, it.n_st, cw, warp, lane); break;
      case 2:  dense_dw_tile<2, BF16>(p, out, it.c0, it.k0, base, full, empty, g, it.n_st, cw, warp, lane); break;
      case 3:  dense_dw_tile<3, BF16>(p, out, it.c0, it.k0, base, full, empty, g, it.n_st, cw, warp, lane); break;
      default: dense_dw_tile<4, BF16>(p, out, it.c0, it.k0, base, full, empty, g, it.n_st, cw, warp, lane); break;
    }
    g += it.n_st;
  }
}

// ---- CUDA-core route ------------------------------------------------------------------------------------------
constexpr int DW_FMA_THREADS = 256, DW_FMA_ROWS = 32;    // rows per shared-memory chunk

// Thread (ty, tx) = (tid / 16, tid % 16) owns rows 4ty..4ty+3 x columns 4tx..4tx+3 of the 64 x 64 tile and adds the
// products row by row with one fmaf each.  The next chunk's loads are in flight while the current one is multiplied.
template <typename T>
__global__ void __launch_bounds__(DW_FMA_THREADS)
fma_dense_dw_kernel(const DenseDwParams p, const T* __restrict__ x, const T* __restrict__ e) {
  __shared__ __align__(16) float xs[DW_FMA_ROWS][DW_FMA_TM];
  __shared__ __align__(16) float es[DW_FMA_ROWS][DW_FMA_TN];
  const int tid = threadIdx.x, tx = tid % 16, ty = tid / 16, lc = tid % 64, lr = tid / 64;
  for (int i = blockIdx.x; i < p.n_items; i += gridDim.x) {
    const int tile = i % p.tiles;
    const long long c0 = (long long)(tile / p.tiles_k) * DW_FMA_TM, k0 = (long long)(tile % p.tiles_k) * DW_FMA_TN;
    const long long r_begin = (long long)(i / p.tiles) * p.seg_stages * DW_STAGE_ROWS;
    long long r_end = r_begin + p.seg_stages * DW_STAGE_ROWS;
    if (r_end > p.N) r_end = p.N;
    const bool cx = c0 + lc < p.C, ce = k0 + lc < p.K;
    float xr[8], er[8];
    auto load = [&](long long n0) {
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        const long long n = n0 + lr + 4 * q;
        xr[q] = (cx && n < r_end) ? to_f32(x[n * p.C + c0 + lc]) : 0.f;
        er[q] = (ce && n < r_end) ? to_f32(e[n * p.K + k0 + lc]) : 0.f;
      }
    };
    float acc[4][4];
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
      for (int b = 0; b < 4; ++b) acc[a][b] = 0.f;
    load(r_begin);
    for (long long n0 = r_begin; n0 < r_end; n0 += DW_FMA_ROWS) {
      __syncthreads();
#pragma unroll
      for (int q = 0; q < 8; ++q) { xs[lr + 4 * q][lc] = xr[q]; es[lr + 4 * q][lc] = er[q]; }
      __syncthreads();
      if (n0 + DW_FMA_ROWS < r_end) load(n0 + DW_FMA_ROWS);
#pragma unroll 8
      for (int r = 0; r < DW_FMA_ROWS; ++r) {
        const float4 a = *reinterpret_cast<const float4*>(&xs[r][4 * ty]);
        const float4 b = *reinterpret_cast<const float4*>(&es[r][4 * tx]);
        const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
        for (int u = 0; u < 4; ++u)
#pragma unroll
          for (int v = 0; v < 4; ++v) acc[u][v] = fmaf(av[u], bv[v], acc[u][v]);
      }
    }
    float* out = p.out + (long long)(i / p.tiles) * p.C * p.K;
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const long long r = c0 + 4 * ty + u;
      if (r >= p.C) break;
#pragma unroll
      for (int v = 0; v < 4; ++v)
        if (k0 + 4 * tx + v < p.K) out[r * p.K + k0 + 4 * tx + v] = acc[u][v];
    }
  }
}

// U[i] = sum over s of ws[s][i], s ascending.
__global__ void __launch_bounds__(256) dense_dw_reduce_kernel(float* __restrict__ u, const float* __restrict__ ws,
                                                              long long CK, int S) {
  const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
  if (i >= CK) return;
  float s = ws[i];
#pragma unroll 4
  for (int j = 1; j < S; ++j) s += ws[(long long)j * CK + i];
  u[i] = s;
}

// Launches the route's kernel and, for S > 1, the reduction.  `tc` selects the wgmma route; the caller has checked
// dense_dw_tc_shape, the pointers' alignment and the device.  N, C, K > 0.
inline int dense_dw_run(bool tc, int dtype, const void* x, const void* e, float* u, long long N, int C, int K,
                        float* workspace, cudaStream_t s) {
  const DwSplit d = dense_dw_split(N, C, K, tc);
  DenseDwParams p;
  p.out = d.S > 1 ? workspace : u;
  p.C = C; p.K = K; p.N = N;
  p.stages = d.stages; p.seg_stages = d.seg_stages;
  p.tiles = (int)d.tiles; p.tiles_k = (int)d.tiles_k; p.n_items = (int)(d.tiles * d.S);
  const int grid = p.n_items < device_info().sm_grid ? p.n_items : device_info().sm_grid;
  const char* name = tc ? "wgmma_dense_dw" : "fma_dense_dw";
  if (tc) {
    DenseDwTmaps maps;
    memset(&maps, 0, sizeof(maps));
    if (int rc = cached_tmap_2d(&maps.x, dtype, x, (uint64_t)C, (uint64_t)N, (uint64_t)C, 64, 64, CU_TENSOR_MAP_SWIZZLE_128B)) return rc;
    if (int rc = cached_tmap_2d(&maps.e, dtype, e, (uint64_t)K, (uint64_t)N, (uint64_t)K, 64, 64, CU_TENSOR_MAP_SWIZZLE_128B)) return rc;
    static thread_local uint64_t configured_h = 0, configured_b = 0;
    if (dtype == BSMM_BF16) {
      if (int rc = ensure_dyn_smem(wgmma_dense_dw_kernel<true>, DwShape::SMEM, configured_b)) return rc;
      wgmma_dense_dw_kernel<true><<<grid, DW_THREADS, DwShape::SMEM, s>>>(p, maps);
    } else {
      if (int rc = ensure_dyn_smem(wgmma_dense_dw_kernel<false>, DwShape::SMEM, configured_h)) return rc;
      wgmma_dense_dw_kernel<false><<<grid, DW_THREADS, DwShape::SMEM, s>>>(p, maps);
    }
  } else {
    BSMM_DISPATCH_DTYPE(dtype, T, {
      fma_dense_dw_kernel<T><<<grid, DW_FMA_THREADS, 0, s>>>(p, static_cast<const T*>(x), static_cast<const T*>(e));
    });
  }
  if (int rc = check_launch(name)) return rc;
  if (d.S > 1) {
    const long long ck = (long long)C * K;
    dense_dw_reduce_kernel<<<(unsigned)((ck + 255) / 256), 256, 0, s>>>(u, workspace, ck, (int)d.S);
    return check_launch(name);
  }
  return 0;
}

}  // namespace bsmm
