// wgmma updat kernel: DW[w] = alpha * sum_p X_p[:, c-blk]^T . DY_p[:, k-blk]  (+ beta * DW[w])
// for 16-bit dtypes, both feature axes, block size 16 / 32 / 64.
//   Replaces hgemm_blocksparse_64x64x64_tn_dds / 32x32x64_tn_dds
//   (reference src/blocksparse_hgemm_nc_op_gpu.cu:553-897) and their Volta parameter-bank hack.
//
// Formulation ("gathered dense GEMM", schedule = blocksparse_b200/lut.py:build_updat_schedule):
//   M axis   = 128 input features = a group of 128/bs consecutive input blocks; consumer warpgroup c owns features
//              64c..64c+63
//   N axis   = the output blocks that have at least one active block in that group, COMPACTED side by side in
//              shared memory (n_act*bs <= 256 columns); every K=16 step is ONE wgmma of N = 64, 128, 192 or 256, the
//              narrowest that holds the kept blocks, so the A slice is read once per step and absent slots cost nothing
//   K axis   = the minibatch (reduction), 64 rows per pipeline stage, 4 wgmma K=16 steps per stage
// Output blocks with nothing to update are neither loaded nor multiplied, and the reference's one-CTA-per-block
// re-read of X and DY becomes one pass per (group, window).  The epilogue writes only the blocks that exist.
//   axis 1: A = X[n][c] (MN-major, two 64-feature boxes), B = DY[n][k] (MN-major, one box per kept block: the slots
//           are the MN atoms of B, BSLOT bytes apart).
//   axis 0: A = X[c][n], B = DY[k][n]: both K-major with 128-byte rows; kept blocks continue the row index.
//
// Warp-specialized and persistent: min(tiles, SMs) CTAs, CTA b runs tiles b, b + gridDim.x, ... (the schedule lists
// them longest first, and lut.py:_balance_windows sizes the windows for exactly this deal).  Warpgroup 0 is the producer:
// one thread streams the stages of all the CTA's tiles through a ring guarded by full / empty mbarriers, running ahead
// into the next tile while the consumers write the previous one out.  Warpgroups 1 and 2 multiply; each consumer warp
// releases a stage as soon as wgmma.wait_group has retired the MMAs that read it.  No CTA-wide barrier after set-up.
#pragma once
#include "common.cuh"
#include "ptx.cuh"

namespace bsmm {

constexpr int UPDAT_THREADS = 3 * 128;  // one producer warpgroup, two consumer warpgroups
constexpr int UPDAT_STAGES = 4;
constexpr int UPDAT_KCHUNK = 64;        // minibatch rows per stage
constexpr int UPDAT_PRODUCER_REGS = 40, UPDAT_CONSUMER_REGS = 232;   // 128 x 40 + 256 x 232 <= 64 K registers
// record layout of lut.py:build_updat_schedule: 64 ints for <= 8 slots per tile (bs 32 / 64), 192 for the 16 slots of bs 16
__host__ __device__ constexpr int updat_rec_ints(int bs) { return bs >= 32 ? 64 : 192; }
__host__ __device__ constexpr int updat_tab_off(int bs) { return bs >= 32 ? 16 : 32; }

struct UpdatTcParams {
  const int32_t* sched;     // build_updat_schedule
  int n_tiles;
  int N;                    // minibatch rows per pair
  int pcount;
  float alpha, beta;
  const float* gate;        // optional, only with gated
  int gated;
  void* dw;
};
struct UpdatTmaps { CUtensorMap x[BSMM_MAX_PAIRS]; CUtensorMap dy[BSMM_MAX_PAIRS]; };

template <int BS> struct UpdatShape {
  static constexpr uint32_t ABYTES = 128 * UPDAT_KCHUNK * 2;     // 16 KB: 128 features
  static constexpr uint32_t BSLOT = BS * UPDAT_KCHUNK * 2;       // one kept output block
  static constexpr uint32_t STAGE = ABYTES + (256 / BS) * BSLOT; // 48 KB
  static constexpr size_t SMEM = UPDAT_STAGES * STAGE + SMEM_ALIGN_SLACK;
};

// One tile of one consumer warpgroup: features 64cw..64cw+63 of the group x NCH*64 compacted columns, reduced over
// the n_chunks stages at ring positions g0, g0 + 1, ...; then its part of the epilogue.
template <int NCH, int BS, bool BF16, bool AXIS0, typename TO>
__device__ __forceinline__ void updat_tile(const UpdatTcParams& p, const int32_t* rec, int n_act, uint32_t base,
                                           uint64_t* full, uint64_t* empty, int g0, int n_chunks, int cw, int warp, int lane) {
  using Sh = UpdatShape<BS>;
  constexpr int ST = UPDAT_STAGES, KT = 256 / BS, TAB = updat_tab_off(BS);
  constexpr uint32_t B_ROW = BS * 2;                  // axis 1: bytes per row of a DY box
  float acc[NCH * 32];
#pragma unroll
  for (int i = 0; i < NCH * 32; ++i) acc[i] = 0.f;

  for (int ch = 0; ch < n_chunks; ++ch) {
    const int g = g0 + ch;
    const uint32_t st = base + (uint32_t)(g % ST) * Sh::STAGE;
    if (!ptx::mbar_wait(&full[g % ST], (uint32_t)(g / ST) & 1)) g_tc_error = 11;
    ptx::wg_fence();
#pragma unroll
    for (int ks = 0; ks < UPDAT_KCHUNK / 16; ++ks) {
      const uint64_t adesc = AXIS0 ? ptx::make_desc(st + cw * (Sh::ABYTES / 2) + ks * 32, 16, 1024, ptx::SWZ_128B)
                                   : ptx::make_desc(st + cw * (Sh::ABYTES / 2) + ks * 2048, Sh::ABYTES / 2, 1024, ptx::SWZ_128B);
      const uint64_t bdesc = AXIS0 ? ptx::make_desc(st + Sh::ABYTES + ks * 32, 16, 1024, ptx::SWZ_128B)
                                   : ptx::make_desc(st + Sh::ABYTES + ks * 16 * B_ROW, Sh::BSLOT, 8 * B_ROW, ptx::swz_for_row(B_ROW));
      ptx::wgmma<BF16, AXIS0 ? 0 : 1, AXIS0 ? 0 : 1, NCH * 64>(acc, adesc, bdesc);
    }
    ptx::wg_commit();
    ptx::wg_wait<1>();                                // the MMAs of the previous stage have retired: hand it back
    if (ch > 0 && lane == 0) ptx::mbar_arrive(&empty[(g - 1) % ST]);
  }
  ptx::wg_wait<0>();
  if (lane == 0) ptx::mbar_arrive(&empty[(g0 + n_chunks - 1) % ST]);
  ptx::wg_fence_regs(acc);

  // epilogue: accumulator (feature row r of the group, column c) -> DW[w][r % BS][c % BS], w from the record's table.
  // Accumulator column 8J + 2(lane % 4) + e sits in acc[4J + 2h + e] (rows r0, r0 + 8), so slot s holds J in
  // [s*BS/8, (s+1)*BS/8).  Both rows lie in one input block (BS >= 16): one table row per thread.
  TO* dw = reinterpret_cast<TO*>(p.dw);
  const int r0 = cw * 64 + warp * 16 + lane / 4;
  const int32_t* wid = rec + TAB + (r0 / BS) * KT;
#pragma unroll
  for (int s = 0; s < NCH * 64 / BS; ++s) {
    if (s >= n_act) break;
    const int w = __ldg(wid + s);
    if (w < 0) continue;
    float g = p.alpha;
    if (p.gated) g *= p.gate[w];
#pragma unroll
    for (int jj = 0; jj < BS / 8; ++jj) {
      const int J = s * (BS / 8) + jj;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float a = acc[4 * J + 2 * h] * g, b = acc[4 * J + 2 * h + 1] * g;
        TO* out = dw + ((size_t)w * BS + (r0 + 8 * h) % BS) * BS + 8 * jj + 2 * (lane % 4);
        if constexpr (sizeof(TO) == 4) {
          float2* o2 = reinterpret_cast<float2*>(out);
          if (p.beta != 0.f) { const float2 old = *o2; a += old.x; b += old.y; }
          *o2 = make_float2(a, b);
        } else {
          uint32_t* o2 = reinterpret_cast<uint32_t*>(out);
          if (p.beta != 0.f) {
            const uint32_t old = *o2;
            if constexpr (BF16) { const __nv_bfloat162 v = *reinterpret_cast<const __nv_bfloat162*>(&old); a += __bfloat162float(v.x); b += __bfloat162float(v.y); }
            else                { const __half2 v = *reinterpret_cast<const __half2*>(&old);        a += __half2float(v.x);     b += __half2float(v.y); }
          }
          *o2 = pack2<BF16>(a, b);
        }
      }
    }
  }
}

template <int BS, bool BF16, bool AXIS0, typename TO>
__global__ void __launch_bounds__(UPDAT_THREADS, 1)
tc_updat_kernel(const __grid_constant__ UpdatTcParams p, const __grid_constant__ UpdatTmaps maps) {
  using Sh = UpdatShape<BS>;
  constexpr int ST = UPDAT_STAGES, KT = 256 / BS, REC = updat_rec_ints(BS);

  extern __shared__ uint8_t smem_raw[];
  __shared__ uint64_t full[ST], empty[ST];
  __shared__ int kcol[KT];                            // producer only: first DY feature of each kept slot
  const uint32_t base = aligned_smem_base(smem_raw);
  const int tid = threadIdx.x, wg = tid / 128;
  const int chunks_per_pair = (p.N + UPDAT_KCHUNK - 1) / UPDAT_KCHUNK;
  const int n_chunks = chunks_per_pair * p.pcount;   // stages per tile

  if (tid == 0) {
    for (int i = 0; i < ST; ++i) {
      ptx::mbar_init(&full[i], 1);
      ptx::mbar_init(&empty[i], 8);                   // one arrival per consumer warp
    }
    ptx::fence_mbar_init();
  }
  __syncthreads();

  if (wg == 0) {
    ptx::setmaxnreg_dec<UPDAT_PRODUCER_REGS>();
    if (tid != 0) return;
    int g = 0;                                        // ring position, continued across the CTA's tiles
    for (int t = blockIdx.x; t < p.n_tiles; t += gridDim.x) {
      const int32_t* rec = p.sched + 4 + (size_t)t * REC;
      const int c0 = __ldg(rec) * BS, n_act = __ldg(rec + 1);
      for (int s = 0; s < n_act; ++s) kcol[s] = __ldg(rec + 8 + s) * BS;
      const uint32_t tx = Sh::ABYTES + (uint32_t)n_act * Sh::BSLOT;
      for (int ch = 0; ch < n_chunks; ++ch, ++g) {
        const int slot = g % ST;
        if (g >= ST && !ptx::mbar_wait(&empty[slot], (uint32_t)(g / ST - 1) & 1)) g_tc_error = 12;
        const uint32_t st = base + (uint32_t)slot * Sh::STAGE;
        uint64_t* bar = &full[slot];
        const int pair = ch / chunks_per_pair;
        const int n0 = (ch % chunks_per_pair) * UPDAT_KCHUNK;
        ptx::mbar_expect_tx(bar, tx);
        if (!AXIS0) {
          ptx::tma_load_2d(st, &maps.x[pair], bar, c0, n0);
          ptx::tma_load_2d(st + Sh::ABYTES / 2, &maps.x[pair], bar, c0 + 64, n0);
          for (int s = 0; s < n_act; ++s) ptx::tma_load_2d(st + Sh::ABYTES + s * Sh::BSLOT, &maps.dy[pair], bar, kcol[s], n0);
        } else {                                      // [128 features][64 n], 128-byte rows
          ptx::tma_load_2d(st, &maps.x[pair], bar, n0, c0);
          for (int s = 0; s < n_act; ++s) ptx::tma_load_2d(st + Sh::ABYTES + s * Sh::BSLOT, &maps.dy[pair], bar, n0, kcol[s]);
        }
      }
    }
    return;
  }

  ptx::setmaxnreg_inc<UPDAT_CONSUMER_REGS>();
  const int cw = wg - 1, warp = (tid / 32) % 4, lane = tid % 32;
  int g = 0;
  for (int t = blockIdx.x; t < p.n_tiles; t += gridDim.x, g += n_chunks) {
    const int32_t* rec = p.sched + 4 + (size_t)t * REC;
    const int n_act = __ldg(rec + 1);
    switch ((n_act * BS + 63) / 64) {                 // MMA width: the 64-column chunks holding kept blocks
      case 1:  updat_tile<1, BS, BF16, AXIS0, TO>(p, rec, n_act, base, full, empty, g, n_chunks, cw, warp, lane); break;
      case 2:  updat_tile<2, BS, BF16, AXIS0, TO>(p, rec, n_act, base, full, empty, g, n_chunks, cw, warp, lane); break;
      case 3:  updat_tile<3, BS, BF16, AXIS0, TO>(p, rec, n_act, base, full, empty, g, n_chunks, cw, warp, lane); break;
      default: updat_tile<4, BS, BF16, AXIS0, TO>(p, rec, n_act, base, full, empty, g, n_chunks, cw, warp, lane); break;
    }
  }
}

template <int BS, bool BF16, bool AXIS0, typename TO>
int launch_tc_updat(const UpdatTcParams& p, const UpdatTmaps& maps, cudaStream_t s) {
  auto kern = tc_updat_kernel<BS, BF16, AXIS0, TO>;
  constexpr size_t smem = UpdatShape<BS>::SMEM;
  static thread_local uint64_t configured = 0;
  if (int e = ensure_dyn_smem(kern, smem, configured)) return e;
  const int grid = p.n_tiles < device_info().sm_grid ? p.n_tiles : device_info().sm_grid;
  kern<<<grid, UPDAT_THREADS, smem, s>>>(p, maps);
  return check_launch(BS == 16 ? "wgmma_updat_bs16" : BS == 32 ? "wgmma_updat_bs32" : "wgmma_updat_bs64");
}

template <int BS, bool BF16, typename TO>
int dispatch_tc_updat(const UpdatTcParams& p, const UpdatTmaps& maps, bool axis0, cudaStream_t s) {
  return axis0 ? launch_tc_updat<BS, BF16, true, TO>(p, maps, s) : launch_tc_updat<BS, BF16, false, TO>(p, maps, s);
}

inline int tc_updat(int dtype, int dw_dtype, int axis, int bsize, int n_c_blocks, int n_k_blocks,
                    const void* const* xs, const void* const* dys, int pcount, void* dw, int N, float alpha,
                    float beta, const float* gate, int gated_dw, const int32_t* sched, int sched_tiles, int sched_tile_blocks,
                    cudaStream_t s) {
  if (dtype != BSMM_F16 && dtype != BSMM_BF16) { fail(0, "fp32 runs on the FMA path"); return TC_NOT_APPLICABLE; }
  if (axis == 0 && (N & 7)) { fail(0, "feature_axis 0 needs N %% 8 == 0 for TMA"); return TC_NOT_APPLICABLE; }
  if (bsize != 16 && bsize != 32 && bsize != 64) { fail(0, "block size %d uses the CUDA-core path", bsize); return TC_NOT_APPLICABLE; }
  if (sched == nullptr || sched_tiles <= 0) { fail(0, "no updat schedule supplied"); return TC_NOT_APPLICABLE; }
  if (sched_tile_blocks != 256 / bsize) return fail(BSMM_E_ARG, "bsmm_updat: schedule built for %d slots per tile, kernel needs %d", sched_tile_blocks, 256 / bsize);
  if (N <= 0) return TC_NOT_APPLICABLE;
  if ((uintptr_t)dw & 15) { fail(0, "dw must be 16-byte aligned"); return TC_NOT_APPLICABLE; }
  for (int i = 0; i < pcount; ++i)
    if (((uintptr_t)xs[i] | (uintptr_t)dys[i]) & 15) { fail(0, "pointers must be 16-byte aligned for TMA"); return TC_NOT_APPLICABLE; }
  if (!wgmma_device()) return TC_NOT_APPLICABLE;

  const uint64_t C = (uint64_t)n_c_blocks * bsize, K = (uint64_t)n_k_blocks * bsize;
  UpdatTmaps maps;
  memset(&maps, 0, sizeof(maps));
  for (int i = 0; i < pcount; ++i) {
    if (axis == 1) {
      if (int e = cached_tmap_2d(&maps.x[i], dtype, xs[i], C, (uint64_t)N, C, 64, UPDAT_KCHUNK, CU_TENSOR_MAP_SWIZZLE_128B)) return e;
      if (int e = cached_tmap_2d(&maps.dy[i], dtype, dys[i], K, (uint64_t)N, K, bsize, UPDAT_KCHUNK, tmap_swizzle_for_row(bsize * 2))) return e;
    } else {       // (features, N): inner dim = minibatch, 64 columns = 128-byte rows
      if (int e = cached_tmap_2d(&maps.x[i], dtype, xs[i], (uint64_t)N, C, (uint64_t)N, UPDAT_KCHUNK, 128, CU_TENSOR_MAP_SWIZZLE_128B)) return e;
      if (int e = cached_tmap_2d(&maps.dy[i], dtype, dys[i], (uint64_t)N, K, (uint64_t)N, UPDAT_KCHUNK, bsize, CU_TENSOR_MAP_SWIZZLE_128B)) return e;
    }
  }
  UpdatTcParams p;
  p.sched = sched; p.n_tiles = sched_tiles; p.N = N; p.pcount = pcount;
  p.alpha = alpha; p.beta = beta; p.gate = gate; p.gated = (gated_dw && gate) ? 1 : 0; p.dw = dw;
  const bool bf = dtype == BSMM_BF16, a0 = axis == 0;
  const bool f32out = dw_dtype == BSMM_F32;
#define BSMM_UPDAT_BS(BSV)                                                                                            \
  if (f32out) return bf ? dispatch_tc_updat<BSV, true, float>(p, maps, a0, s)                            \
                        : dispatch_tc_updat<BSV, false, float>(p, maps, a0, s);                          \
  return bf ? dispatch_tc_updat<BSV, true, __nv_bfloat16>(p, maps, a0, s)                                \
            : dispatch_tc_updat<BSV, false, __half>(p, maps, a0, s);
  if (bsize == 16) { BSMM_UPDAT_BS(16) }
  if (bsize == 32) { BSMM_UPDAT_BS(32) }
  BSMM_UPDAT_BS(64)
#undef BSMM_UPDAT_BS
}

}  // namespace bsmm
