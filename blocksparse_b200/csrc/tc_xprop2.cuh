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
constexpr int XP2_REC = 8;           // ints per merged entry: (input block, W block of output 0..3 or -1, pad)

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

// sched: lut.py:build_wide_schedule in device memory: tile offsets at int32 index 2, merged entries at ent_off.
inline int tc_xprop2(int dtype, int axis, int bprop, int n_out, int n_in, int blocks, const void* x, const void* w, void* y,
                     int N, const int32_t* sched, int n_tiles, int variant, int ent_off, cudaStream_t s) {
  if (dtype != BSMM_F16 && dtype != BSMM_BF16) return fail(BSMM_E_ARG, "bsmm_xprop: the wide-tile schedule needs a 16-bit dtype");
  if (variant < 1 || variant > 3) return fail(BSMM_E_ARG, "bsmm_xprop: wide-tile variant %d (1..3)", variant);
  const int tb = variant == 3 ? 4 : 2;
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
    default: return bf ? dispatch_tc_xprop2<4, 2, true>(p, maps, n_tiles, a0, bp, s) : dispatch_tc_xprop2<4, 2, false>(p, maps, n_tiles, a0, bp, s);
  }
}

}  // namespace bsmm
