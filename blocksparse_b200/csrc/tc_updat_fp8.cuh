// fp8 updat kernel: DW[w] = sum_p scale_p * XT_p[c-blk] . DYT_p[k-blk]^T  (+ DW[w] when beta = 1),
// scale_p = x_scale_inv_p * dy_scale_inv_p, for e4m3 / e5m2 operands, block size 32 / 64 (DESIGN.md "fp8 updat").
//
// Formulation: tc_updat_kernel's gathered dense GEMM (csrc/tc_updat.cuh) on its feature-axis-0 operand path, with the
// same schedule (lut.py:build_updat_schedule) and the same persistent, warp-specialized layout: warpgroup 0 produces,
// one thread streaming stages through a full / empty mbarrier ring; warpgroups 1 and 2 multiply 64 features each.
// fp8 wgmma takes K-major operands only, so both operands are feature-major copies with the minibatch contiguous:
//   A = XT[c][n]  (128 features of the group),   B = DYT[k][n]  (the tile's kept output blocks, stacked)
// A stage holds 128 minibatch rows: one 128-byte swizzle span of 1-byte rows, four m64nNk32 steps. Each stage belongs
// to one (x, dy) pair; TMA zero-fills rows past N, so N needs no alignment, only the pitch does.
//
// Accumulation: Hopper's fp8 MMA keeps fewer accumulator bits than fp32 (DESIGN.md 6e), so each stage's four k32 steps
// accumulate in a fragment that starts from zero (scale-d = 0 on the first step); after wgmma.wait the fragment is
// multiplied by scale_p and added to an fp32 total on CUDA cores (one fma per element), stage by stage in schedule
// order. A 256-column tile runs as two halves of at most 128 columns, so a consumer holds at most a 128-float total and
// a 64-float fragment. No atomics: each tile belongs to one CTA and results are bitwise reproducible.
#pragma once
#include <type_traits>
#include "tc.cuh"
#include "tc_updat.cuh"

namespace bsmm {

constexpr int UPDAT8_KCHUNK = 128;      // minibatch rows per stage: one 128-byte row of 1-byte elements

struct UpdatFp8Params {
  const int32_t* sched;                 // build_updat_schedule (256 / bs slots per tile)
  int n_tiles;
  int chunks_per_pair;                  // ceil(N / 128)
  int pcount;
  int beta;                             // 0 or 1
  void* dw;
  const float* x_scale_inv[BSMM_MAX_PAIRS];
  const float* dy_scale_inv[BSMM_MAX_PAIRS];
};

template <int BS> struct Updat8Shape {
  static constexpr uint32_t ABYTES = 128 * UPDAT8_KCHUNK;         // 16 KB: 128 features x 128 rows
  static constexpr uint32_t BSLOT = BS * UPDAT8_KCHUNK;           // one kept output block
  static constexpr uint32_t STAGE = ABYTES + (256 / BS) * BSLOT;  // 48 KB, as the 16-bit kernel's
  static constexpr size_t SMEM = UPDAT_STAGES * STAGE + SMEM_ALIGN_SLACK;
};

// The four k32 steps of one stage for the NC 64-column chunks starting at column 64 * c0, into a zeroed fragment that
// is then scaled and added to tot[32 * c0 ..]. Accumulator layout as in ptx.cuh: the fragment's element i is the
// total's element 32 * c0 + i.
template <int NC, int XT, int DT>
__device__ __forceinline__ void updat8_half(float* tot, int c0, uint32_t a_base, uint32_t b_base, float sc) {
  float f[NC * 32];
  ptx::wg_fence();
#pragma unroll
  for (int ks = 0; ks < UPDAT8_KCHUNK / 32; ++ks) {
    const uint64_t adesc = ptx::make_desc(a_base + ks * 32, 16, 1024, ptx::SWZ_128B);
    const uint64_t bdesc = ptx::make_desc(b_base + c0 * 64 * 128 + ks * 32, 16, 1024, ptx::SWZ_128B);
    ptx::wgmma_fp8<XT, DT, NC * 64>(f, adesc, bdesc, ks > 0);
  }
  ptx::wg_commit();
  ptx::wg_wait<0>();
  ptx::wg_fence_regs(f);
#pragma unroll
  for (int i = 0; i < NC * 32; ++i) tot[c0 * 32 + i] = __fmaf_rn(f[i], sc, tot[c0 * 32 + i]);
}

template <int NCH, int BS, int XT, int DT, typename TO>
__device__ __forceinline__ void updat8_tile(const UpdatFp8Params& p, const int32_t* rec, int n_act, uint32_t base,
                                            uint64_t* full, uint64_t* empty, int g0, int n_chunks, int cw, int warp,
                                            int lane) {
  using Sh = Updat8Shape<BS>;
  constexpr int ST = UPDAT_STAGES, KT = 256 / BS, TAB = updat_tab_off(BS);
  constexpr int H0 = NCH < 2 ? NCH : 2, H1 = NCH - H0;          // 64-column chunks in each half
  float tot[NCH * 32];
#pragma unroll
  for (int i = 0; i < NCH * 32; ++i) tot[i] = 0.f;

  for (int ch = 0; ch < n_chunks; ++ch) {
    const int g = g0 + ch, pair = ch / p.chunks_per_pair;
    const float sc = __fmul_rn(__ldg(p.x_scale_inv[pair]), __ldg(p.dy_scale_inv[pair]));
    const uint32_t st = base + (uint32_t)(g % ST) * Sh::STAGE;
    if (!ptx::mbar_wait(&full[g % ST], (uint32_t)(g / ST) & 1)) g_tc_error = 13;
    const uint32_t a_base = st + cw * (Sh::ABYTES / 2), b_base = st + Sh::ABYTES;
    updat8_half<H0, XT, DT>(tot, 0, a_base, b_base, sc);
    if constexpr (H1 > 0) updat8_half<H1, XT, DT>(tot, H0, a_base, b_base, sc);
    if (lane == 0) ptx::mbar_arrive(&empty[g % ST]);             // this warp's MMAs on the stage have retired
  }

  // epilogue: total (feature row r of the group, column c) -> DW[w][r % BS][c % BS], w from the record's table, as in
  // tc_updat.cuh's updat_tile
  constexpr bool BF16 = std::is_same<TO, __nv_bfloat16>::value;
  TO* dw = reinterpret_cast<TO*>(p.dw);
  const int r0 = cw * 64 + warp * 16 + lane / 4;
  const int32_t* wid = rec + TAB + (r0 / BS) * KT;
#pragma unroll
  for (int s = 0; s < NCH * 64 / BS; ++s) {
    if (s >= n_act) break;
    const int w = __ldg(wid + s);
    if (w < 0) continue;
#pragma unroll
    for (int jj = 0; jj < BS / 8; ++jj) {
      const int J = s * (BS / 8) + jj;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float a = tot[4 * J + 2 * h], b = tot[4 * J + 2 * h + 1];
        TO* out = dw + ((size_t)w * BS + (r0 + 8 * h) % BS) * BS + 8 * jj + 2 * (lane % 4);
        if constexpr (sizeof(TO) == 4) {
          float2* o2 = reinterpret_cast<float2*>(out);
          if (p.beta) { const float2 old = *o2; a += old.x; b += old.y; }
          *o2 = make_float2(a, b);
        } else {
          uint32_t* o2 = reinterpret_cast<uint32_t*>(out);
          if (p.beta) {
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

// XT / DT: 0 = e4m3, 1 = e5m2
template <int BS, int XT, int DT, typename TO>
__global__ void __launch_bounds__(UPDAT_THREADS, 1)
tc_updat_fp8_kernel(const __grid_constant__ UpdatFp8Params p, const __grid_constant__ UpdatTmaps maps) {
  using Sh = Updat8Shape<BS>;
  constexpr int ST = UPDAT_STAGES, KT = 256 / BS, REC = updat_rec_ints(BS);

  extern __shared__ uint8_t smem_raw[];
  __shared__ uint64_t full[ST], empty[ST];
  __shared__ int kcol[KT];                            // producer only: first DY feature of each kept slot
  const uint32_t base = aligned_smem_base(smem_raw);
  const int tid = threadIdx.x, wg = tid / 128;
  const int n_chunks = p.chunks_per_pair * p.pcount; // stages per tile

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
        if (g >= ST && !ptx::mbar_wait(&empty[slot], (uint32_t)(g / ST - 1) & 1)) g_tc_error = 14;
        const uint32_t st = base + (uint32_t)slot * Sh::STAGE;
        uint64_t* bar = &full[slot];
        const int pair = ch / p.chunks_per_pair;
        const int n0 = (ch % p.chunks_per_pair) * UPDAT8_KCHUNK;
        ptx::mbar_expect_tx(bar, tx);
        ptx::tma_load_2d(st, &maps.x[pair], bar, n0, c0);                               // [128 features][128 n]
        for (int s = 0; s < n_act; ++s) ptx::tma_load_2d(st + Sh::ABYTES + s * Sh::BSLOT, &maps.dy[pair], bar, n0, kcol[s]);
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
    switch ((n_act * BS + 63) / 64) {                 // the 64-column chunks holding kept blocks
      case 1:  updat8_tile<1, BS, XT, DT, TO>(p, rec, n_act, base, full, empty, g, n_chunks, cw, warp, lane); break;
      case 2:  updat8_tile<2, BS, XT, DT, TO>(p, rec, n_act, base, full, empty, g, n_chunks, cw, warp, lane); break;
      case 3:  updat8_tile<3, BS, XT, DT, TO>(p, rec, n_act, base, full, empty, g, n_chunks, cw, warp, lane); break;
      default: updat8_tile<4, BS, XT, DT, TO>(p, rec, n_act, base, full, empty, g, n_chunks, cw, warp, lane); break;
    }
  }
}

template <int BS, int XT, int DT, typename TO>
int launch_tc_updat_fp8(const UpdatFp8Params& p, const UpdatTmaps& maps, cudaStream_t s) {
  auto kern = tc_updat_fp8_kernel<BS, XT, DT, TO>;
  constexpr size_t smem = Updat8Shape<BS>::SMEM;
  static thread_local uint64_t configured = 0;
  if (int e = ensure_dyn_smem(kern, smem, configured)) return e;
  const int grid = p.n_tiles < device_info().sm_grid ? p.n_tiles : device_info().sm_grid;
  kern<<<grid, UPDAT_THREADS, smem, s>>>(p, maps);
  return check_launch(BS == 32 ? "wgmma_updat_fp8_bs32" : "wgmma_updat_fp8_bs64");
}

template <int BS, int XT, int DT>
int dispatch_tc_updat_fp8(const UpdatFp8Params& p, const UpdatTmaps& maps, int dw_dtype, cudaStream_t s) {
  if (dw_dtype == BSMM_F32) return launch_tc_updat_fp8<BS, XT, DT, float>(p, maps, s);
  if (dw_dtype == BSMM_BF16) return launch_tc_updat_fp8<BS, XT, DT, __nv_bfloat16>(p, maps, s);
  return launch_tc_updat_fp8<BS, XT, DT, __half>(p, maps, s);
}

template <int BS>
int dispatch_tc_updat_fp8(const UpdatFp8Params& p, const UpdatTmaps& maps, int x_dtype, int dy_dtype, int dw_dtype,
                          cudaStream_t s) {
  const bool x5 = x_dtype == BSMM_E5M2, d5 = dy_dtype == BSMM_E5M2;
  if (x5) return d5 ? dispatch_tc_updat_fp8<BS, 1, 1>(p, maps, dw_dtype, s) : dispatch_tc_updat_fp8<BS, 1, 0>(p, maps, dw_dtype, s);
  return d5 ? dispatch_tc_updat_fp8<BS, 0, 1>(p, maps, dw_dtype, s) : dispatch_tc_updat_fp8<BS, 0, 0>(p, maps, dw_dtype, s);
}

// Arguments already checked by bsmm_updat_fp8: bsize 32 / 64, fp8 xt and dyt, fp32 / fp16 / bf16 dw, pcount in range,
// non-null aligned pointers, 0 < N <= pitch < 2^31, pitch % 16 == 0, the schedule's slot count.
inline int tc_updat_fp8(int x_dtype, int dy_dtype, int dw_dtype, int bsize, int n_c_blocks, int n_k_blocks,
                        const void* const* xts, const void* const* dyts, const float* const* x_scale_invs,
                        const float* const* dy_scale_invs, int pcount, void* dw, long long N, long long pitch, int beta,
                        const int32_t* sched, int sched_tiles, cudaStream_t s) {
  if (!wgmma_device()) return fail(BSMM_E_NODEV, "bsmm_updat_fp8: %s", err_buf());
  const uint64_t C = (uint64_t)n_c_blocks * bsize, K = (uint64_t)n_k_blocks * bsize;
  UpdatTmaps maps;
  memset(&maps, 0, sizeof(maps));
  UpdatFp8Params p;
  memset(&p, 0, sizeof(p));
  for (int i = 0; i < pcount; ++i) {                  // (features, N) with rows `pitch` bytes apart, 128-byte boxes
    if (int e = cached_tmap_2d(&maps.x[i], x_dtype, xts[i], (uint64_t)N, C, (uint64_t)pitch, UPDAT8_KCHUNK, 128, CU_TENSOR_MAP_SWIZZLE_128B)) return e;
    if (int e = cached_tmap_2d(&maps.dy[i], dy_dtype, dyts[i], (uint64_t)N, K, (uint64_t)pitch, UPDAT8_KCHUNK, bsize, CU_TENSOR_MAP_SWIZZLE_128B)) return e;
    p.x_scale_inv[i] = x_scale_invs[i];
    p.dy_scale_inv[i] = dy_scale_invs[i];
  }
  p.sched = sched; p.n_tiles = sched_tiles; p.chunks_per_pair = (int)((N + UPDAT8_KCHUNK - 1) / UPDAT8_KCHUNK);
  p.pcount = pcount; p.beta = beta; p.dw = dw;
  return bsize == 32 ? dispatch_tc_updat_fp8<32>(p, maps, x_dtype, dy_dtype, dw_dtype, s)
                     : dispatch_tc_updat_fp8<64>(p, maps, x_dtype, dy_dtype, dw_dtype, s);
}

}  // namespace bsmm
