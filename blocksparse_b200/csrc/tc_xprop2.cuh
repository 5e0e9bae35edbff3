// wgmma xprop over WIDE output tiles: block-sparse fprop / bprop for 16-bit dtypes and 32 x 32 blocks, both feature axes.
//   Replaces hgemm_blocksparse_64x32x32_nx_dsd (reference src/blocksparse_hgemm_nc_op_gpu.cu:38-551) and the
//   feature-axis-0 family hgemm_blocksparse_xn_64_sdd (src/blocksparse_hgemm_cn_64_op_gpu.cu:9-717).
//
// What differs from csrc/tc.cuh (one output block per CTA): a CTA owns TB = 2 or 4 consecutive output blocks and walks
// the MERGED LUT rows of the tile (lut.py:build_wide_schedule): one entry per input block that any of them consumes,
// carrying the TB W blocks (absent ones are read from beyond the end of the weight tensor, which TMA fills with zeros).
// Each activation tile is therefore staged once for up to TB output blocks instead of once per block, and every K=16
// step is one MMA of N = TB*32 instead of TB MMAs of N = 32.  The price is multiplying the zero blocks of the tile.
// Opt-in (BlocksparseMatMul, BSMM_XPROP2=1..3); variants (blocks per tile, m64 row groups per CTA):
//   1 = (2, 1)  64 minibatch rows per CTA: more CTAs for small minibatches
//   2 = (2, 2)  128 rows
//   3 = (4, 2)  128 rows, 128 output features
// Accumulation order is the merged entry order (ascending input block), so results are deterministic.
#pragma once
#include "tc.cuh"

namespace bsmm {

template <int TB, int MI> struct Xp2Shape {
  static constexpr uint32_t XBYTES = MI * 64 * 32 * 2;                    // MI*64 minibatch rows x 32 features
  static constexpr uint32_t WBYTES = 32 * 32 * 2;
  static constexpr uint32_t STAGE = (XBYTES + TB * WBYTES + 1023) / 1024 * 1024;
  static constexpr size_t SMEM = XP_STAGES * STAGE + SMEM_ALIGN_SLACK;
};
constexpr int XP2_REC = 16;          // ints per merged entry: (input block, W block of output 0..7 or -1, pad)

struct Xprop2Params {
  const int32_t* tile_off;   // [n_tiles + 1] first merged entry of every tile
  const int32_t* ent;        // [entries][XP2_REC]
  int n_out;
  int w_absent;              // W block index whose TMA box lies wholly out of bounds (= number of blocks): zeros
  void* y;
  long long y_pitch;         // elements
  int N;
};

template <int TB, int MI, bool BF16, bool AXIS0, bool BPROP>
__global__ void __launch_bounds__(XP_THREADS)
tc_xprop2_kernel(const Xprop2Params p, const __grid_constant__ XpropTmaps maps) {
  using Sh = Xp2Shape<TB, MI>;
  constexpr int ST = XP_STAGES, NW = TB * 32;
  extern __shared__ uint8_t smem_raw[];
  __shared__ uint64_t full[ST];
  const uint32_t base = aligned_smem_base(smem_raw);
  const int tid = threadIdx.x, warp = tid / 32, lane = tid % 32;
  const int nt = blockIdx.x, t = blockIdx.y;
  const int first = p.tile_off[t], count = p.tile_off[t + 1] - first;
  const int32_t* ent = p.ent + (size_t)first * XP2_REC;

  auto issue = [&](int e) {                                // one thread: stage merged entry e
    const int32_t* r = ent + e * XP2_REC;
    const uint32_t st = base + (uint32_t)(e % ST) * Sh::STAGE;
    uint64_t* bar = &full[e % ST];
    ptx::mbar_expect_tx(bar, Sh::XBYTES + TB * Sh::WBYTES);
    if (!AXIS0) {
      ptx::tma_load_2d(st, &maps.x, bar, r[0] * 32, nt * MI * 64);                       // [MI*64 n][32 c]
    } else {
#pragma unroll
      for (int m = 0; m < MI; ++m) ptx::tma_load_2d(st + m * 4096, &maps.x, bar, nt * MI * 64 + m * 64, r[0] * 32);
    }
#pragma unroll
    for (int j = 0; j < TB; ++j) {
      const int wb = r[1 + j];
      ptx::tma_load_2d(st + Sh::XBYTES + j * Sh::WBYTES, &maps.w, bar, 0, (wb < 0 ? p.w_absent : wb) * 32);
    }
  };

  if (tid == 0) {
    for (int i = 0; i < ST; ++i) ptx::mbar_init(&full[i], 1);
    ptx::fence_mbar_init();
    ptx::prefetch_tensormap(&maps.x); ptx::prefetch_tensormap(&maps.w);
  }
  __syncthreads();
  if (tid == 0)
    for (int e = 0; e < count && e < ST; ++e) issue(e);

  float acc[MI][NW / 2];
#pragma unroll
  for (int m = 0; m < MI; ++m)
#pragma unroll
    for (int i = 0; i < NW / 2; ++i) acc[m][i] = 0.f;

  for (int e = 0; e < count; ++e) {
    const uint32_t st = base + (uint32_t)(e % ST) * Sh::STAGE;
    if (!ptx::mbar_wait(&full[e % ST], (uint32_t)(e / ST) & 1)) g_tc_error = 41;
    ptx::wg_fence();
#pragma unroll
    for (int ks = 0; ks < 2; ++ks) {
      // fprop: the TB W blocks are TB MN atoms of 32 columns, one block apart (LBO); bprop: their rows simply continue
      const uint64_t bdesc = BPROP ? ptx::make_desc(st + Sh::XBYTES + ks * 32, 16, 512, ptx::SWZ_64B)
                                   : ptx::make_desc(st + Sh::XBYTES + ks * 1024, Sh::WBYTES, 512, ptx::SWZ_64B);
#pragma unroll
      for (int m = 0; m < MI; ++m) {
        const uint64_t adesc = AXIS0 ? ptx::make_desc(st + m * 4096 + ks * 2048, 4096, 1024, ptx::SWZ_128B)
                                     : ptx::make_desc(st + m * 64 * 64 + ks * 32, 16, 512, ptx::SWZ_64B);
        ptx::wgmma<BF16, AXIS0 ? 1 : 0, BPROP ? 0 : 1, NW>(acc[m], adesc, bdesc);
      }
    }
    ptx::wg_commit();
    ptx::wg_wait<1>();
    __syncthreads();
    if (tid == 0 && e >= 1 && e - 1 + ST < count) issue(e - 1 + ST);
  }
  ptx::wg_wait<0>();
#pragma unroll
  for (int m = 0; m < MI; ++m) ptx::wg_fence_regs(acc[m]);

  // epilogue (output blocks with no entry are written as zeros)
  uint16_t* y = reinterpret_cast<uint16_t*>(p.y);
#pragma unroll
  for (int m = 0; m < MI; ++m)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const long long n = (long long)nt * MI * 64 + m * 64 + warp * 16 + lane / 4 + 8 * h;
      if (n >= p.N) continue;
#pragma unroll
      for (int j = 0; j < NW / 8; ++j) {
        const int cl = 8 * j + 2 * (lane % 4);
        const int o = t * TB + cl / 32;
        if (o >= p.n_out) continue;
        const int col = o * 32 + cl % 32;
        const float a = acc[m][4 * j + 2 * h], b = acc[m][4 * j + 2 * h + 1];
        if (!AXIS0) {
          *reinterpret_cast<uint32_t*>(y + n * p.y_pitch + col) = pack2<BF16>(a, b);
        } else {
          y[(long long)col * p.y_pitch + n] = pack1<BF16>(a);
          y[(long long)(col + 1) * p.y_pitch + n] = pack1<BF16>(b);
        }
      }
    }
}

template <int TB, int MI, bool BF16, bool AXIS0, bool BPROP>
int launch_tc_xprop2(const Xprop2Params& p, const XpropTmaps& maps, int n_tiles, cudaStream_t s) {
  auto kern = tc_xprop2_kernel<TB, MI, BF16, AXIS0, BPROP>;
  constexpr size_t smem = Xp2Shape<TB, MI>::SMEM;
  static thread_local uint64_t configured = 0;
  if (int e = ensure_dyn_smem(kern, smem, configured)) return e;
  kern<<<dim3((unsigned)((p.N + MI * 64 - 1) / (MI * 64)), (unsigned)n_tiles), XP_THREADS, smem, s>>>(p, maps);
  return check_launch("wgmma_xprop2_bs32");
}

template <int TB, int MI, bool BF16>
int dispatch_tc_xprop2(const Xprop2Params& p, const XpropTmaps& maps, int n_tiles, bool axis0, bool bprop, cudaStream_t s) {
  if (axis0) return bprop ? launch_tc_xprop2<TB, MI, BF16, true, true>(p, maps, n_tiles, s) : launch_tc_xprop2<TB, MI, BF16, true, false>(p, maps, n_tiles, s);
  return bprop ? launch_tc_xprop2<TB, MI, BF16, false, true>(p, maps, n_tiles, s) : launch_tc_xprop2<TB, MI, BF16, false, false>(p, maps, n_tiles, s);
}

// ---- grouped tiles: the default for 32 x 32 blocks when lut.py:pick_xprop_tile selects them ---------------------------
// A CTA owns 128 minibatch rows x G consecutive output blocks and walks the same merged entries, but only the W blocks
// that exist are fetched (block j of the tile always lands in slot j of the stage; the slot of an absent block keeps
// stale bytes that nothing reads) and only they are multiplied: one m64n32k16 MMA per K = 16 step into the 16
// accumulator registers of block j.  Every output element therefore sees exactly the MMAs of tc_xprop_kernel in the same
// (ascending input block) order, so results are bit-identical to it and an output depends on no block its LUT row does
// not list.  One warpgroup owns both 64-row halves: 32 G accumulator registers per thread, three CTAs per SM at G = 4.
template <int G> struct XpgShape {
  static constexpr uint32_t XBYTES = 128 * 32 * 2;
  static constexpr uint32_t WBYTES = 32 * 32 * 2;
  static constexpr uint32_t STAGE = XBYTES + G * WBYTES;
  static constexpr size_t SMEM = XP_STAGES * STAGE + SMEM_ALIGN_SLACK;
};

// Merged entries whose records a CTA keeps in shared memory at a time.  The loop below is lock-step (wait, multiply,
// CTA barrier, refill), so a record read from global memory by the refilling thread would put an L2 round trip into
// every iteration; the records of up to XPG_LUT entries are copied to shared memory first, and a longer tile drains
// its pipeline once per XPG_LUT entries to load the next ones.
constexpr int XPG_LUT = 128;

template <int G, bool BF16, bool AXIS0, bool BPROP>
__global__ void __launch_bounds__(XP_THREADS)
tc_xprop_grouped_kernel(const Xprop2Params p, const __grid_constant__ XpropTmaps maps, const int n_tiles) {
  using Sh = XpgShape<G>;
  constexpr int ST = XP_STAGES;
  extern __shared__ uint8_t smem_raw[];
  __shared__ uint64_t full[ST];
  const uint32_t base = aligned_smem_base(smem_raw);
  const int tid = threadIdx.x, warp = tid / 32, lane = tid % 32;
  // the output tiles of one minibatch tile are neighbours in the grid, so CTAs that run together share activation tiles
  // in L2 (with the minibatch tile running fastest an activation tensor larger than L2 is streamed once per output tile)
  const int nt = blockIdx.x / n_tiles, t = blockIdx.x % n_tiles;
  const int first = p.tile_off[t], count = p.tile_off[t + 1] - first;
  const int32_t* ent = p.ent + (size_t)first * XP2_REC;
  // per entry of the current chunk: input block, W block of output 0..G-1 (or -1), mask of the blocks that exist
  __shared__ int32_t rec[XPG_LUT][G + 2];

  auto issue = [&](int c0, int e) {                        // one thread: stage merged entry c0 + e (e: index in the chunk)
    const int32_t* r = rec[e];
    const int g = c0 + e;
    const uint32_t st = base + (uint32_t)(g % ST) * Sh::STAGE;
    uint64_t* bar = &full[g % ST];
    const uint32_t mask = (uint32_t)r[G + 1];
    ptx::mbar_expect_tx(bar, Sh::XBYTES + (uint32_t)__popc(mask) * Sh::WBYTES);
    const int c = r[0];
    if (!AXIS0) {
      ptx::tma_load_2d(st, &maps.x, bar, c * 32, nt * 128);                              // [128 n][32 c]
    } else {                                                                             // [32 c][128 n] as two 64-column boxes
      ptx::tma_load_2d(st, &maps.x, bar, nt * 128, c * 32);
      ptx::tma_load_2d(st + Sh::XBYTES / 2, &maps.x, bar, nt * 128 + 64, c * 32);
    }
#pragma unroll
    for (int j = 0; j < G; ++j)
      if (mask >> j & 1) ptx::tma_load_2d(st + Sh::XBYTES + j * Sh::WBYTES, &maps.w, bar, 0, r[1 + j] * 32);
  };

  if (tid == 0) {
    for (int i = 0; i < ST; ++i) ptx::mbar_init(&full[i], 1);
    ptx::fence_mbar_init();
    ptx::prefetch_tensormap(&maps.x); ptx::prefetch_tensormap(&maps.w);
  }

  float acc[2][G][16];
#pragma unroll
  for (int m = 0; m < 2; ++m)
#pragma unroll
    for (int j = 0; j < G; ++j)
#pragma unroll
      for (int i = 0; i < 16; ++i) acc[m][j][i] = 0.f;

  for (int c0 = 0; c0 < count; c0 += XPG_LUT) {
    const int n = min(count - c0, XPG_LUT);
    __syncthreads();                                         // barriers initialized; the previous chunk is consumed and its records are free
    for (int i = tid; i < n; i += XP_THREADS) {
      const int32_t* r = ent + (size_t)(c0 + i) * XP2_REC;
      int32_t mask = 0;
      rec[i][0] = __ldg(r);
#pragma unroll
      for (int j = 0; j < G; ++j) {
        const int32_t wb = __ldg(r + 1 + j);
        rec[i][1 + j] = wb;
        mask |= (int32_t)(wb >= 0) << j;
      }
      rec[i][G + 1] = mask;
    }
    __syncthreads();
    if (tid == 0)
      for (int e = 0; e < n && e < ST; ++e) issue(c0, e);
    for (int e = 0; e < n; ++e) {
      const int g = c0 + e;
      const uint32_t st = base + (uint32_t)(g % ST) * Sh::STAGE;
      const uint32_t mask = (uint32_t)rec[e][G + 1];         // uniform over the CTA
      if (!ptx::mbar_wait(&full[g % ST], (uint32_t)(g / ST) & 1)) g_tc_error = 45;
      ptx::wg_fence();
#pragma unroll
      for (int j = 0; j < G; ++j) {
        if (mask >> j & 1) {
#pragma unroll
          for (int ks = 0; ks < 2; ++ks) {                   // descriptors as tc_xprop_kernel<32>: fprop reads W MN-major, bprop K-major
            const uint32_t wb = st + Sh::XBYTES + j * Sh::WBYTES;
            const uint64_t bdesc = BPROP ? ptx::make_desc(wb + ks * 32, 16, 512, ptx::SWZ_64B)
                                         : ptx::make_desc(wb + ks * 1024, Sh::WBYTES, 512, ptx::SWZ_64B);
#pragma unroll
            for (int m = 0; m < 2; ++m) {
              const uint64_t adesc = AXIS0 ? ptx::make_desc(st + m * (Sh::XBYTES / 2) + ks * 2048, Sh::XBYTES / 2, 1024, ptx::SWZ_128B)
                                           : ptx::make_desc(st + m * 64 * 64 + ks * 32, 16, 512, ptx::SWZ_64B);
              ptx::wgmma<BF16, AXIS0 ? 1 : 0, BPROP ? 0 : 1, 32>(acc[m][j], adesc, bdesc);
            }
          }
        }
      }
      ptx::wg_commit();
      ptx::wg_wait<1>();                                     // entry e-1 has been consumed by the whole warpgroup ...
      __syncthreads();
      if (tid == 0 && e >= 1 && e - 1 + ST < n) issue(c0, e - 1 + ST);   // ... so its buffer can be refilled
    }
    ptx::wg_wait<0>();
  }
#pragma unroll
  for (int m = 0; m < 2; ++m)
#pragma unroll
    for (int j = 0; j < G; ++j) ptx::wg_fence_regs(acc[m][j]);

  // epilogue (output blocks with no entry are written as zeros)
  uint16_t* y = reinterpret_cast<uint16_t*>(p.y);
#pragma unroll
  for (int m = 0; m < 2; ++m)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const long long n = (long long)nt * 128 + m * 64 + warp * 16 + lane / 4 + 8 * h;
      if (n >= p.N) continue;
#pragma unroll
      for (int j = 0; j < G; ++j) {
        const int o = t * G + j;
        if (o >= p.n_out) continue;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const int col = o * 32 + 8 * q + 2 * (lane % 4);
          const float a = acc[m][j][4 * q + 2 * h], b = acc[m][j][4 * q + 2 * h + 1];
          if (!AXIS0) {
            *reinterpret_cast<uint32_t*>(y + n * p.y_pitch + col) = pack2<BF16>(a, b);
          } else {
            y[(long long)col * p.y_pitch + n] = pack1<BF16>(a);
            y[(long long)(col + 1) * p.y_pitch + n] = pack1<BF16>(b);
          }
        }
      }
    }
}

template <int G, bool BF16, bool AXIS0, bool BPROP>
int launch_tc_xprop_grouped(const Xprop2Params& p, const XpropTmaps& maps, int n_tiles, cudaStream_t s) {
  auto kern = tc_xprop_grouped_kernel<G, BF16, AXIS0, BPROP>;
  constexpr size_t smem = XpgShape<G>::SMEM;
  static thread_local uint64_t configured = 0;
  if (int e = ensure_dyn_smem(kern, smem, configured)) return e;
  const long long ctas = (long long)((p.N + 127) / 128) * n_tiles;
  if (ctas > 0x7fffffffLL) return fail(BSMM_E_LIMIT, "bsmm_xprop: %lld CTAs exceed the grid limit", ctas);
  kern<<<dim3((unsigned)ctas), XP_THREADS, smem, s>>>(p, maps, n_tiles);
  return check_launch("wgmma_xprop_bs32");                 // the default 32 x 32 route keeps one name whatever tile it runs
}

template <int G, bool BF16>
int dispatch_tc_xprop_grouped(const Xprop2Params& p, const XpropTmaps& maps, int n_tiles, bool axis0, bool bprop, cudaStream_t s) {
  if (axis0) return bprop ? launch_tc_xprop_grouped<G, BF16, true, true>(p, maps, n_tiles, s) : launch_tc_xprop_grouped<G, BF16, true, false>(p, maps, n_tiles, s);
  return bprop ? launch_tc_xprop_grouped<G, BF16, false, true>(p, maps, n_tiles, s) : launch_tc_xprop_grouped<G, BF16, false, false>(p, maps, n_tiles, s);
}

// variant 4: the grouped kernel with G = 4 output blocks per CTA.
// sched: lut.py:build_wide_schedule in device memory: tile offsets at int32 index 2, merged entries at ent_off.
inline int tc_xprop2(int dtype, int axis, int bprop, int n_out, int n_in, int blocks, const void* x, const void* w, void* y,
                     int N, const int32_t* sched, int n_tiles, int variant, int ent_off, cudaStream_t s) {
  if (dtype != BSMM_F16 && dtype != BSMM_BF16) return fail(BSMM_E_ARG, "bsmm_xprop: the wide-tile schedule needs a 16-bit dtype");
  if (variant < 1 || variant > 4) return fail(BSMM_E_ARG, "bsmm_xprop: wide-tile variant %d (1..4)", variant);
  const int tb = variant >= 3 ? 4 : 2;
  if (sched == nullptr || n_tiles <= 0 || (long long)n_tiles * tb < n_out || ent_off < n_tiles + 3)
    return fail(BSMM_E_ARG, "bsmm_xprop: inconsistent wide-tile schedule (tiles=%d variant=%d entries at %d)", n_tiles, variant, ent_off);
  if (axis == 0 && (N & 7)) { fail(0, "feature_axis 0 needs N %% 8 == 0 for TMA (row pitch multiple of 16 bytes)"); return TC_NOT_APPLICABLE; }
  if (((uintptr_t)x | (uintptr_t)w | (uintptr_t)y) & 15) { fail(0, "pointers must be 16-byte aligned for TMA"); return TC_NOT_APPLICABLE; }
  if (!wgmma_device()) return TC_NOT_APPLICABLE;

  const int rows = variant == 1 ? 64 : 128;
  const uint64_t Cin = (uint64_t)n_in * 32, Cout = (uint64_t)n_out * 32;
  XpropTmaps maps;
  if (axis == 1) {
    if (int e = cached_tmap_2d(&maps.x, dtype, x, Cin, (uint64_t)N, Cin, 32, rows, CU_TENSOR_MAP_SWIZZLE_64B)) return e;
  } else {
    if (int e = cached_tmap_2d(&maps.x, dtype, x, (uint64_t)N, Cin, (uint64_t)N, 64, 32, CU_TENSOR_MAP_SWIZZLE_128B)) return e;
  }
  if (int e = cached_tmap_2d(&maps.w, dtype, w, 32, (uint64_t)blocks * 32, 32, 32, 32, CU_TENSOR_MAP_SWIZZLE_64B)) return e;
  Xprop2Params p;
  p.tile_off = sched + 2; p.ent = sched + ent_off; p.n_out = n_out; p.w_absent = blocks;
  p.y = y; p.y_pitch = axis == 0 ? (long long)N : (long long)Cout; p.N = N;
  const bool bf = dtype == BSMM_BF16, a0 = axis == 0, bp = bprop != 0;
  switch (variant) {
    case 1: return bf ? dispatch_tc_xprop2<2, 1, true>(p, maps, n_tiles, a0, bp, s) : dispatch_tc_xprop2<2, 1, false>(p, maps, n_tiles, a0, bp, s);
    case 2: return bf ? dispatch_tc_xprop2<2, 2, true>(p, maps, n_tiles, a0, bp, s) : dispatch_tc_xprop2<2, 2, false>(p, maps, n_tiles, a0, bp, s);
    case 3: return bf ? dispatch_tc_xprop2<4, 2, true>(p, maps, n_tiles, a0, bp, s) : dispatch_tc_xprop2<4, 2, false>(p, maps, n_tiles, a0, bp, s);
    default: return bf ? dispatch_tc_xprop_grouped<4, true>(p, maps, n_tiles, a0, bp, s) : dispatch_tc_xprop_grouped<4, false>(p, maps, n_tiles, a0, bp, s);
  }
}

}  // namespace bsmm
