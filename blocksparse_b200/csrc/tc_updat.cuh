// wgmma updat kernel: DW[w] = alpha * sum_p X_p[:, c-blk]^T . DY_p[:, k-blk]  (+ beta * DW[w])
// for 16-bit dtypes, both feature axes, block size 16 / 32 / 64.
//   Replaces hgemm_blocksparse_64x64x64_tn_dds / 32x32x64_tn_dds
//   (reference src/blocksparse_hgemm_nc_op_gpu.cu:553-897) and their Volta parameter-bank hack.
//
// Formulation ("gathered dense GEMM", schedule = blocksparse_b200/lut.py:build_updat_schedule):
//   M axis   = 128 input features = a group of 128/bs consecutive input blocks; warpgroup g owns features 64g..64g+63
//   N axis   = the output blocks that have at least one active block in that group, COMPACTED side by side in
//              shared memory (n_act*bs <= 256 columns, multiplied in 64-column wgmma chunks: absent slots cost nothing)
//   K axis   = the minibatch (reduction), 64 rows per pipeline stage, 4 wgmma K=16 steps per stage
// Output blocks with nothing to update are neither loaded nor multiplied, and the reference's one-CTA-per-block
// re-read of X and DY becomes one pass per (group, window).  The epilogue writes only the blocks that exist.
//   axis 1: A = X[n][c] (MN-major, two 64-feature boxes), B = DY[n][k] (MN-major, one box per kept block).
//   axis 0: A = X[c][n], B = DY[k][n]: both K-major with 128-byte rows; kept blocks continue the row index.
#pragma once
#include "common.cuh"
#include "ptx.cuh"

namespace bsmm {

constexpr int UPDAT_THREADS = 2 * 128;  // two warpgroups
constexpr int UPDAT_STAGES = 4;
constexpr int UPDAT_KCHUNK = 64;        // minibatch rows per stage
// record layout of lut.py:build_updat_schedule: 64 ints for <= 8 slots per tile (bs 32 / 64), 192 for the 16 slots of bs 16
__host__ __device__ constexpr int updat_rec_ints(int bs) { return bs >= 32 ? 64 : 192; }
__host__ __device__ constexpr int updat_tab_off(int bs) { return bs >= 32 ? 16 : 32; }

struct UpdatTcParams {
  const int32_t* sched;     // build_updat_schedule
  int N;                    // minibatch rows per pair
  int pcount;
  float alpha, beta;
  const float* gate;        // optional, only with gated
  int gated;
  void* dw;
};
struct UpdatTmaps { CUtensorMap x[BSMM_MAX_PAIRS]; CUtensorMap dy[BSMM_MAX_PAIRS]; };

template <int BS>
constexpr size_t updat_smem_bytes() {
  return (size_t)UPDAT_STAGES * (128 * UPDAT_KCHUNK * 2 + 256 * UPDAT_KCHUNK * 2) + SMEM_ALIGN_SLACK;
}

template <int BS, bool BF16, bool AXIS0, typename TO>
__global__ void __launch_bounds__(UPDAT_THREADS, 1)
tc_updat_kernel(const UpdatTcParams p, const __grid_constant__ UpdatTmaps maps) {
  constexpr int ST = UPDAT_STAGES;
  constexpr int KT = 256 / BS;                        // slots per tile
  constexpr uint32_t ABYTES = 128 * UPDAT_KCHUNK * 2; // 16 KB
  constexpr uint32_t BSLOT = BS * UPDAT_KCHUNK * 2;   // one kept output block
  constexpr uint32_t STAGE_BYTES = ABYTES + KT * BSLOT;
  constexpr uint32_t B_ROW = BS * 2;                  // axis 1: bytes per row of a DY box
  constexpr int REC = updat_rec_ints(BS), TAB = updat_tab_off(BS);

  extern __shared__ uint8_t smem_raw[];
  __shared__ uint64_t full[ST];
  __shared__ int rec[REC];
  const uint32_t base = aligned_smem_base(smem_raw);
  const int tid = threadIdx.x, warp = tid / 32, lane = tid % 32, wg = warp / 4;
  const int chunks_per_pair = (p.N + UPDAT_KCHUNK - 1) / UPDAT_KCHUNK;
  const int n_chunks = chunks_per_pair * p.pcount;

  for (int i = tid; i < REC; i += UPDAT_THREADS) rec[i] = p.sched[4 + (size_t)blockIdx.x * REC + i];
  if (tid == 0) {
    for (int i = 0; i < ST; ++i) ptx::mbar_init(&full[i], 1);
    ptx::fence_mbar_init();
  }
  __syncthreads();
  const int c0 = rec[0], n_act = rec[1];
  const int nch = (n_act * BS + 63) / 64;             // 64-column wgmma chunks holding kept blocks

  auto issue = [&](int ch) {                          // one thread: stage minibatch chunk ch
    const uint32_t st = base + (uint32_t)(ch % ST) * STAGE_BYTES;
    uint64_t* bar = &full[ch % ST];
    const int pair = ch / chunks_per_pair;
    const int n0 = (ch % chunks_per_pair) * UPDAT_KCHUNK;
    ptx::mbar_expect_tx(bar, ABYTES + (uint32_t)n_act * BSLOT);
    if (!AXIS0) {
      ptx::tma_load_2d(st, &maps.x[pair], bar, c0 * BS, n0);
      ptx::tma_load_2d(st + ABYTES / 2, &maps.x[pair], bar, c0 * BS + 64, n0);
      for (int s = 0; s < n_act; ++s) ptx::tma_load_2d(st + ABYTES + s * BSLOT, &maps.dy[pair], bar, rec[8 + s] * BS, n0);
    } else {                                          // [128 features][64 n], 128-byte rows
      ptx::tma_load_2d(st, &maps.x[pair], bar, n0, c0 * BS);
      for (int s = 0; s < n_act; ++s) ptx::tma_load_2d(st + ABYTES + s * BSLOT, &maps.dy[pair], bar, n0, rec[8 + s] * BS);
    }
  };
  if (tid == 0)
    for (int ch = 0; ch < n_chunks && ch < ST; ++ch) issue(ch);

  float acc[4][32];
#pragma unroll
  for (int q = 0; q < 4; ++q)
#pragma unroll
    for (int i = 0; i < 32; ++i) acc[q][i] = 0.f;

  for (int ch = 0; ch < n_chunks; ++ch) {
    const uint32_t st = base + (uint32_t)(ch % ST) * STAGE_BYTES;
    if (!ptx::mbar_wait(&full[ch % ST], (uint32_t)(ch / ST) & 1)) g_tc_error = 11;
    ptx::wg_fence();
#pragma unroll
    for (int ks = 0; ks < UPDAT_KCHUNK / 16; ++ks) {
      const uint64_t adesc = AXIS0 ? ptx::make_desc(st + wg * (ABYTES / 2) + ks * 32, 16, 1024, ptx::SWZ_128B)
                                   : ptx::make_desc(st + wg * (ABYTES / 2) + ks * 2048, ABYTES / 2, 1024, ptx::SWZ_128B);
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        if (q < nch) {                                // uniform across the CTA
          const uint32_t b0 = st + ABYTES + q * 8192;  // 64 columns = 64 rows of 128 bytes (axis 0) or 64/BS slots (axis 1)
          const uint64_t bdesc = AXIS0 ? ptx::make_desc(b0 + ks * 32, 16, 1024, ptx::SWZ_128B)
                                       : ptx::make_desc(b0 + ks * 16 * B_ROW, BSLOT, 8 * B_ROW, ptx::swz_for_row(B_ROW));
          if (AXIS0) ptx::wgmma_n64<BF16, 0, 0>(acc[q], adesc, bdesc);
          else       ptx::wgmma_n64<BF16, 1, 1>(acc[q], adesc, bdesc);
        }
      }
    }
    ptx::wg_commit();
    ptx::wg_wait<1>();
    __syncthreads();
    if (tid == 0 && ch >= 1 && ch - 1 + ST < n_chunks) issue(ch - 1 + ST);
  }
  ptx::wg_wait<0>();
#pragma unroll
  for (int q = 0; q < 4; ++q) ptx::wg_fence_regs(acc[q]);

  // epilogue: accumulator (feature row r of the group, column c) -> DW[w][r % BS][c % BS], w from the record's table
  TO* dw = reinterpret_cast<TO*>(p.dw);
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    if (q >= nch) continue;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int col = q * 64 + 8 * j + 2 * (lane % 4);
      const int s = col / BS, jj = col % BS;
      if (s >= n_act) continue;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int r = wg * 64 + (warp % 4) * 16 + lane / 4 + 8 * h;
        const int w = rec[TAB + (r / BS) * KT + s];
        if (w < 0) continue;
        float g = p.alpha;
        if (p.gated) g *= p.gate[w];
        float a = acc[q][4 * j + 2 * h] * g, b = acc[q][4 * j + 2 * h + 1] * g;
        TO* out = dw + ((size_t)w * BS + r % BS) * BS + jj;
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
int launch_tc_updat(const UpdatTcParams& p, const UpdatTmaps& maps, int n_tiles, cudaStream_t s) {
  auto kern = tc_updat_kernel<BS, BF16, AXIS0, TO>;
  constexpr size_t smem = updat_smem_bytes<BS>();
  static thread_local uint64_t configured = 0;
  if (int e = ensure_dyn_smem(kern, smem, configured)) return e;
  kern<<<n_tiles, UPDAT_THREADS, smem, s>>>(p, maps);
  return check_launch(BS == 16 ? "wgmma_updat_bs16" : BS == 32 ? "wgmma_updat_bs32" : "wgmma_updat_bs64");
}

template <int BS, bool BF16, typename TO>
int dispatch_tc_updat(const UpdatTcParams& p, const UpdatTmaps& maps, int n_tiles, bool axis0, cudaStream_t s) {
  return axis0 ? launch_tc_updat<BS, BF16, true, TO>(p, maps, n_tiles, s) : launch_tc_updat<BS, BF16, false, TO>(p, maps, n_tiles, s);
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
  p.sched = sched; p.N = N; p.pcount = pcount;
  p.alpha = alpha; p.beta = beta; p.gate = gate; p.gated = (gated_dw && gate) ? 1 : 0; p.dw = dw;
  const bool bf = dtype == BSMM_BF16, a0 = axis == 0;
  const bool f32out = dw_dtype == BSMM_F32;
#define BSMM_UPDAT_BS(BSV)                                                                                            \
  if (f32out) return bf ? dispatch_tc_updat<BSV, true, float>(p, maps, sched_tiles, a0, s)                            \
                        : dispatch_tc_updat<BSV, false, float>(p, maps, sched_tiles, a0, s);                          \
  return bf ? dispatch_tc_updat<BSV, true, __nv_bfloat16>(p, maps, sched_tiles, a0, s)                                \
            : dispatch_tc_updat<BSV, false, __half>(p, maps, sched_tiles, a0, s);
  if (bsize == 16) { BSMM_UPDAT_BS(16) }
  if (bsize == 32) { BSMM_UPDAT_BS(32) }
  BSMM_UPDAT_BS(64)
#undef BSMM_UPDAT_BS
}

}  // namespace bsmm
