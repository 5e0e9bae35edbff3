// fp8 block-sparse fprop / bprop on wgmma (sm_90a), with the per-tensor quantisation that feeds it.
//
// Quantisation (bsmm_fp8_quantize, bsmm_fp8_weights; the exact contract is in include/bsmm_b200.h):
//   fp8_amax      amax = max |x|, as an atomicMax on the bits of |x| (non-negative floats order like their bits, and
//                 every NaN sorts above +inf), so the result is exact and independent of the order of the blocks.
//   fp8_quantize  y = cvt.rn.satfinite(x * s), s = FP8_MAX / amax; block 0 also stores scale_inv = amax / FP8_MAX.
//   fp8_weights   the same cast over a (blocks, bs, bs) weight tensor, one CTA per block, writing the block as stored
//                 and transposed.
//   fp8_quantize_t (bsmm_fp8_quantize_t) the same cast over a (rows, cols) tensor in 64 x 64 tiles, writing it as
//                 stored and / or transposed with a padded pitch: the feature-major operands of the fp8 updat
//                 (csrc/tc_updat_fp8.cuh).
//
// xprop (DESIGN.md "fp8 fprop / bprop"): tc_xprop_kernel's formulation (csrc/tc.cuh) with 1-byte operands. One CTA (one
// warpgroup) owns one output block of 128 minibatch rows and walks its LUT row in order, TMA staging each entry's
// activation tile [128 n][bs] and weight block [bs][bs] into a ring of shared-memory stages, one mbarrier each.
// fp8 wgmma has no transposed operands, so both are K-major: A is the activation tile; B is a wq_t block (fprop: rows
// are output features k, columns input features c) or a wq block (bprop: rows c, columns k) -- the same descriptor
// either way. One m64n{bs}k32 wgmma per 32 features and 64-row half.
// Accumulation: Hopper's fp8 MMA is reported to keep fewer accumulator bits than fp32, so each LUT entry's product is
// summed by wgmma into a fragment it starts from zero (scale-d = 0 on the entry's first K step), and the fragment is
// then added to an fp32 total on CUDA cores, in LUT order. No atomics anywhere: results are bitwise reproducible.
#pragma once
#include <cuda_fp8.h>
#include "tc.cuh"

namespace bsmm {

inline bool fp8_code(int dt) { return dt == BSMM_E4M3 || dt == BSMM_E5M2; }

// ---- quantisation -----------------------------------------------------------------------------------------------
template <int FMT> __device__ __forceinline__ float fp8_max() { return FMT == BSMM_E5M2 ? 57344.f : 448.f; }
// two fp32 -> two fp8 (a in the low byte), round to nearest even, saturating finite values; NaN -> 0x7f
template <int FMT> __device__ __forceinline__ uint16_t fp8x2(float a, float b) {
  return (uint16_t)__nv_cvt_float2_to_fp8x2(make_float2(a, b), __NV_SATFINITE, FMT == BSMM_E5M2 ? __NV_E5M2 : __NV_E4M3);
}
template <int FMT> __device__ __forceinline__ uint8_t fp8x1(float a) {
  return (uint8_t)__nv_cvt_float_to_fp8(a, __NV_SATFINITE, FMT == BSMM_E5M2 ? __NV_E5M2 : __NV_E4M3);
}
template <int FMT> __device__ __forceinline__ float fp8_scale(float amax) {
  return amax == 0.f ? 1.f : __fdiv_rn(fp8_max<FMT>(), amax);
}
template <int FMT> __device__ __forceinline__ float fp8_scale_inv(float amax) {
  if (amax == 0.f) return 1.f;
  return isfinite(amax) ? __fdiv_rn(amax, fp8_max<FMT>()) : __int_as_float(0x7fffffff);
}
template <typename T> __device__ __forceinline__ uint32_t abs_bits(T v) { return __float_as_uint(to_f32<T>(v)) & 0x7fffffffu; }

constexpr int FP8_THREADS = 256;
constexpr int FP8_MAX_CTAS = 2048;

template <typename T>
__global__ void __launch_bounds__(FP8_THREADS) fp8_amax_kernel(const T* __restrict__ x, long long n, bool vec,
                                                                unsigned int* amax_bits) {
  constexpr int V = 16 / sizeof(T);
  const long long tid = (long long)blockIdx.x * FP8_THREADS + threadIdx.x, stride = (long long)gridDim.x * FP8_THREADS;
  const long long nv = vec ? n / V : 0;
  uint32_t m = 0;
  for (long long i = tid; i < nv; i += stride) {
    const uint4 u = __ldg(reinterpret_cast<const uint4*>(x) + i);
    const T* e = reinterpret_cast<const T*>(&u);
#pragma unroll
    for (int j = 0; j < V; ++j) m = max(m, abs_bits(e[j]));
  }
  for (long long i = nv * V + tid; i < n; i += stride) m = max(m, abs_bits(x[i]));
  m = __reduce_max_sync(0xffffffffu, m);
  __shared__ uint32_t part[FP8_THREADS / 32];
  if (threadIdx.x % 32 == 0) part[threadIdx.x / 32] = m;
  __syncthreads();
  if (threadIdx.x < 32) {
    m = threadIdx.x < FP8_THREADS / 32 ? part[threadIdx.x] : 0u;
    m = __reduce_max_sync(0xffffffffu, m);
    if (threadIdx.x == 0) atomicMax(amax_bits, m);
  }
}

template <typename T, int FMT>
__global__ void __launch_bounds__(FP8_THREADS) fp8_quantize_kernel(const T* __restrict__ x, long long n, bool vec,
                                                                    const float* amax, float* scale_inv, uint8_t* y) {
  constexpr int V = 16 / sizeof(T);
  const float a = *amax, s = fp8_scale<FMT>(a);
  if (blockIdx.x == 0 && threadIdx.x == 0) *scale_inv = fp8_scale_inv<FMT>(a);
  const long long tid = (long long)blockIdx.x * FP8_THREADS + threadIdx.x, stride = (long long)gridDim.x * FP8_THREADS;
  const long long nv = vec ? n / V : 0;
  for (long long i = tid; i < nv; i += stride) {
    const uint4 u = __ldg(reinterpret_cast<const uint4*>(x) + i);
    const T* e = reinterpret_cast<const T*>(&u);
    uint16_t q[V / 2];
#pragma unroll
    for (int j = 0; j < V / 2; ++j)
      q[j] = fp8x2<FMT>(__fmul_rn(to_f32<T>(e[2 * j]), s), __fmul_rn(to_f32<T>(e[2 * j + 1]), s));
    if constexpr (V == 8)
      reinterpret_cast<uint2*>(y)[i] = make_uint2(q[0] | (uint32_t)q[1] << 16, q[2] | (uint32_t)q[3] << 16);
    else
      reinterpret_cast<uint32_t*>(y)[i] = q[0] | (uint32_t)q[1] << 16;
  }
  for (long long i = nv * V + tid; i < n; i += stride) y[i] = fp8x1<FMT>(__fmul_rn(to_f32<T>(x[i]), s));
}

// One CTA per weight block: wq[b] = the block cast as stored (2 elements per cvt), wq_t[b] = its transpose, assembled
// 4 bytes at a time from a shared-memory copy.
template <typename T, int FMT, int BS>
__global__ void __launch_bounds__(FP8_THREADS) fp8_weights_kernel(const T* __restrict__ w, const float* amax,
                                                                   float* scale_inv, uint8_t* wq, uint8_t* wq_t) {
  __shared__ uint8_t t[BS][BS + 4];
  const float a = *amax, s = fp8_scale<FMT>(a);
  if (blockIdx.x == 0 && threadIdx.x == 0) *scale_inv = fp8_scale_inv<FMT>(a);
  const long long off = (long long)blockIdx.x * BS * BS;
  for (int i = threadIdx.x; i < BS * BS / 2; i += FP8_THREADS) {
    const int r = 2 * i / BS, c = 2 * i % BS;
    const uint16_t q = fp8x2<FMT>(__fmul_rn(to_f32<T>(w[off + 2 * i]), s), __fmul_rn(to_f32<T>(w[off + 2 * i + 1]), s));
    reinterpret_cast<uint16_t*>(wq + off)[i] = q;
    t[r][c] = (uint8_t)q; t[r][c + 1] = (uint8_t)(q >> 8);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < BS * BS / 4; i += FP8_THREADS) {
    const int k = 4 * i / BS, c = 4 * i % BS;                // wq_t[k][c .. c + 3] = wq[c .. c + 3][k]
    reinterpret_cast<uint32_t*>(wq_t + off)[i] =
        t[c][k] | (uint32_t)t[c + 1][k] << 8 | (uint32_t)t[c + 2][k] << 16 | (uint32_t)t[c + 3][k] << 24;
  }
}

// The cast of fp8_quantize over a (rows, cols) tensor in 64 x 64 tiles, writing y (rows x cols, as fp8_quantize does)
// and / or yt[c][r] (cols x pitch, zero in [rows, pitch)). Each tile goes through shared memory as t[c][r], so the
// loads of x, the stores of y and the 4-byte stores of yt all run along rows. Codes are those of fp8_quantize: the
// same fp32 product and the same per-element conversion.
constexpr int FP8T_TILE = 64;
template <typename T, int FMT>
__global__ void __launch_bounds__(FP8_THREADS) fp8_quantize_t_kernel(const T* __restrict__ x, long long rows, long long cols,
                                                                      const float* amax, float* scale_inv, uint8_t* y,
                                                                      uint8_t* yt, long long pitch, long long row_tiles,
                                                                      long long tiles) {
  constexpr int TL = FP8T_TILE;
  __shared__ __align__(4) uint8_t t[TL][TL + 4];
  const float a = *amax, s = fp8_scale<FMT>(a);
  if (blockIdx.x == 0 && threadIdx.x == 0) *scale_inv = fp8_scale_inv<FMT>(a);
  for (long long tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
    const long long r0 = (tile % row_tiles) * TL, c0 = (tile / row_tiles) * TL;
    for (int i = threadIdx.x; i < TL * TL; i += FP8_THREADS) {
      const int r = i / TL, c = i % TL;
      const long long gr = r0 + r, gc = c0 + c;
      uint8_t q = 0;
      if (gr < rows && gc < cols) {
        q = fp8x1<FMT>(__fmul_rn(to_f32<T>(x[gr * cols + gc]), s));
        if (y) y[gr * cols + gc] = q;
      }
      t[c][r] = q;
    }
    __syncthreads();
    if (yt)
      for (int i = threadIdx.x; i < TL * TL / 4; i += FP8_THREADS) {
        const int c = i / (TL / 4), r = 4 * (i % (TL / 4));
        const long long gc = c0 + c, gr = r0 + r;                // pitch % 16 == 0: gr < pitch covers gr + 3 too
        if (gc < cols && gr < pitch) *reinterpret_cast<uint32_t*>(yt + gc * pitch + gr) = *reinterpret_cast<const uint32_t*>(&t[c][r]);
      }
    __syncthreads();
  }
}

template <typename T>
inline int launch_fp8_amax(const T* x, long long n, float* amax, cudaStream_t s) {
  cudaError_t e = cudaMemsetAsync(amax, 0, sizeof(float), s);
  if (e != cudaSuccess) { cudaGetLastError(); return fail((int)e, "fp8_amax: %s", cudaGetErrorString(e)); }
  if (n == 0) return 0;
  constexpr int V = 16 / sizeof(T);
  const bool vec = ((uintptr_t)x & 15) == 0;
  const long long per_cta = (long long)FP8_THREADS * V * 4;
  const long long ctas = (n + per_cta - 1) / per_cta;
  const unsigned grid = (unsigned)(ctas < FP8_MAX_CTAS ? ctas : FP8_MAX_CTAS);
  fp8_amax_kernel<T><<<grid, FP8_THREADS, 0, s>>>(x, n, vec, reinterpret_cast<unsigned int*>(amax));
  return check_launch("fp8_amax");
}

template <typename T, int FMT>
inline int launch_fp8_quantize(const T* x, long long n, float* amax, float* scale_inv, uint8_t* y, cudaStream_t s) {
  if (int e = launch_fp8_amax<T>(x, n, amax, s)) return e;
  constexpr int V = 16 / sizeof(T);
  const bool vec = ((uintptr_t)x & 15) == 0 && ((uintptr_t)y & (V - 1)) == 0;
  const long long per_cta = (long long)FP8_THREADS * V * 4;
  const long long ctas = (n + per_cta - 1) / per_cta;      // n = 0: one CTA, which only stores scale_inv = 1
  const unsigned grid = (unsigned)(ctas < 1 ? 1 : ctas < FP8_MAX_CTAS ? ctas : FP8_MAX_CTAS);
  fp8_quantize_kernel<T, FMT><<<grid, FP8_THREADS, 0, s>>>(x, n, vec, amax, scale_inv, y);
  return check_launch("fp8_quantize");
}

template <typename T, int FMT>
inline int launch_fp8_quantize_t(const T* x, long long rows, long long cols, float* amax, float* scale_inv, uint8_t* y,
                                 uint8_t* yt, long long pitch, cudaStream_t s) {
  if (int e = launch_fp8_amax<T>(x, rows * cols, amax, s)) return e;
  const long long span = yt && pitch > rows ? pitch : rows;      // yt's zero pad lies in rows [rows, pitch)
  const long long row_tiles = (span + FP8T_TILE - 1) / FP8T_TILE, col_tiles = (cols + FP8T_TILE - 1) / FP8T_TILE;
  const long long tiles = row_tiles * col_tiles;
  const unsigned grid = (unsigned)(tiles < 1 ? 1 : tiles < 8 * FP8_MAX_CTAS ? tiles : 8 * FP8_MAX_CTAS);  // tiles = 0: scale_inv only
  fp8_quantize_t_kernel<T, FMT><<<grid, FP8_THREADS, 0, s>>>(x, rows, cols, amax, scale_inv, y, yt, pitch,
                                                              row_tiles > 0 ? row_tiles : 1, tiles);
  return check_launch("fp8_quantize_t");
}

template <typename T, int FMT>
inline int launch_fp8_weights(int bsize, int blocks, const T* w, float* amax, float* scale_inv, uint8_t* wq, uint8_t* wq_t,
                              cudaStream_t s) {
  if (int e = launch_fp8_amax<T>(w, (long long)blocks * bsize * bsize, amax, s)) return e;
  if (bsize == 32) fp8_weights_kernel<T, FMT, 32><<<blocks, FP8_THREADS, 0, s>>>(w, amax, scale_inv, wq, wq_t);
  else fp8_weights_kernel<T, FMT, 64><<<blocks, FP8_THREADS, 0, s>>>(w, amax, scale_inv, wq, wq_t);
  return check_launch("fp8_weights");
}

// ---- xprop --------------------------------------------------------------------------------------------------------
constexpr int XP8_STAGES = 8;         // twice tc_xprop's ring: each stage holds half the bytes
template <int BS> struct Xprop8Shape {
  static constexpr uint32_t XBYTES = 128 * BS;                              // activation tile: 128 minibatch rows x BS features
  static constexpr uint32_t WBYTES = BS * BS;
  static constexpr uint32_t STAGE = (XBYTES + WBYTES + 1023) / 1024 * 1024;
  static constexpr size_t SMEM = XP8_STAGES * STAGE + SMEM_ALIGN_SLACK;
};

struct XpropFp8Params {
  const int32_t* lut;        // row LUT: [n_out][2] = (first entry, count), entries (W block, input block)
  void* y;
  long long y_pitch;         // elements
  int N;
  const float* x_scale_inv;
  const float* w_scale_inv;
};

// XT / WT: 0 = e4m3, 1 = e5m2
template <int BS, int XT, int WT, bool BF16>
__global__ void __launch_bounds__(XP_THREADS)
tc_xprop_fp8_kernel(const XpropFp8Params p, const __grid_constant__ XpropTmaps maps) {
  using Sh = Xprop8Shape<BS>;
  constexpr int ST = XP8_STAGES;
  constexpr uint32_t ROW = BS;                             // bytes per row of a W block / activation tile
  constexpr uint32_t SWZ = ptx::swz_for_row(ROW);
  extern __shared__ uint8_t smem_raw[];
  __shared__ uint64_t full[ST];
  const uint32_t base = aligned_smem_base(smem_raw);
  const int tid = threadIdx.x, warp = tid / 32, lane = tid % 32;
  const int nt = blockIdx.x, o = blockIdx.y;
  const int first = p.lut[2 * o], count = p.lut[2 * o + 1];
  const int2* ent = reinterpret_cast<const int2*>(p.lut) + first;

  auto issue = [&](int e) {                                // one thread: stage entry e
    const int2 wi = ent[e];                                // (W block, input block)
    const uint32_t st = base + (uint32_t)(e % ST) * Sh::STAGE;
    uint64_t* bar = &full[e % ST];
    ptx::mbar_expect_tx(bar, Sh::XBYTES + Sh::WBYTES);
    ptx::tma_load_2d(st, &maps.x, bar, wi.y * BS, nt * 128);                  // [128 n][BS c]
    ptx::tma_load_2d(st + Sh::XBYTES, &maps.w, bar, 0, wi.x * BS);            // [BS out][BS in]
  };

  if (tid == 0) {
    for (int i = 0; i < ST; ++i) ptx::mbar_init(&full[i], 1);
    ptx::fence_mbar_init();
    ptx::prefetch_tensormap(&maps.x); ptx::prefetch_tensormap(&maps.w);
  }
  __syncthreads();
  if (tid == 0)
    for (int e = 0; e < count && e < ST; ++e) issue(e);

  float tot[2][BS / 2], f[2][BS / 2];
#pragma unroll
  for (int m = 0; m < 2; ++m)
#pragma unroll
    for (int i = 0; i < BS / 2; ++i) tot[m][i] = f[m][i] = 0.f;

  for (int e = 0; e < count; ++e) {
    const uint32_t st = base + (uint32_t)(e % ST) * Sh::STAGE;
    if (!ptx::mbar_wait(&full[e % ST], (uint32_t)(e / ST) & 1)) g_tc_error = 1;
    ptx::wg_fence();
#pragma unroll
    for (int ks = 0; ks < BS / 32; ++ks) {                 // entry e's product into f, starting from zero
      const uint64_t bdesc = ptx::make_desc(st + Sh::XBYTES + ks * 32, 16, 8 * ROW, SWZ);
#pragma unroll
      for (int m = 0; m < 2; ++m) {
        const uint64_t adesc = ptx::make_desc(st + m * 64 * ROW + ks * 32, 16, 8 * ROW, SWZ);
        ptx::wgmma_fp8<XT, WT, BS>(f[m], adesc, bdesc, ks > 0);
      }
    }
    ptx::wg_commit();
    // The fragment is read as soon as its MMAs finish. ptxas serialises every wgmma of a kernel in which CUDA-core code
    // reads one fragment while another fragment's MMAs are in flight (C7514), so the add does not overlap this CTA's
    // next MMAs; the other CTAs on the SM keep the tensor cores busy meanwhile.
    ptx::wg_wait<0>();
    ptx::wg_fence_regs(f[0]);
    ptx::wg_fence_regs(f[1]);
#pragma unroll
    for (int m = 0; m < 2; ++m)
#pragma unroll
      for (int i = 0; i < BS / 2; ++i) tot[m][i] += f[m][i];
    __syncthreads();                                       // the whole warpgroup is done with stage e ...
    if (tid == 0 && e + ST < count) issue(e + ST);         // ... so it can be refilled
  }

  // epilogue: one fp32 scale, one rounding (an empty LUT row has count 0 and writes zeros)
  const float sc = count > 0 ? __fmul_rn(*p.x_scale_inv, *p.w_scale_inv) : 0.f;
  uint16_t* y = reinterpret_cast<uint16_t*>(p.y);
#pragma unroll
  for (int m = 0; m < 2; ++m)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const long long n = (long long)nt * 128 + m * 64 + warp * 16 + lane / 4 + 8 * h;
      if (n >= p.N) continue;
#pragma unroll
      for (int j = 0; j < BS / 8; ++j) {
        const int col = o * BS + 8 * j + 2 * (lane % 4);
        const float a = __fmul_rn(tot[m][4 * j + 2 * h], sc), b = __fmul_rn(tot[m][4 * j + 2 * h + 1], sc);
        *reinterpret_cast<uint32_t*>(y + n * p.y_pitch + col) = pack2<BF16>(a, b);
      }
    }
}

template <int BS, int XT, int WT, bool BF16>
int launch_tc_xprop_fp8(const XpropFp8Params& p, const XpropTmaps& maps, int n_out, cudaStream_t s) {
  auto kern = tc_xprop_fp8_kernel<BS, XT, WT, BF16>;
  constexpr size_t smem = Xprop8Shape<BS>::SMEM;
  static thread_local uint64_t configured = 0;
  if (int e = ensure_dyn_smem(kern, smem, configured)) return e;
  kern<<<dim3((unsigned)((p.N + 127) / 128), (unsigned)n_out), XP_THREADS, smem, s>>>(p, maps);
  return check_launch(BS == 32 ? "wgmma_xprop_fp8_bs32" : "wgmma_xprop_fp8_bs64");
}

template <int BS, int XT, int WT>
int dispatch_tc_xprop_fp8(const XpropFp8Params& p, const XpropTmaps& maps, int n_out, bool bf16, cudaStream_t s) {
  return bf16 ? launch_tc_xprop_fp8<BS, XT, WT, true>(p, maps, n_out, s) : launch_tc_xprop_fp8<BS, XT, WT, false>(p, maps, n_out, s);
}

template <int BS>
int dispatch_tc_xprop_fp8(const XpropFp8Params& p, const XpropTmaps& maps, int n_out, int x_dtype, int w_dtype, bool bf16,
                          cudaStream_t s) {
  const bool x5 = x_dtype == BSMM_E5M2, w5 = w_dtype == BSMM_E5M2;
  if (x5) return w5 ? dispatch_tc_xprop_fp8<BS, 1, 1>(p, maps, n_out, bf16, s) : dispatch_tc_xprop_fp8<BS, 1, 0>(p, maps, n_out, bf16, s);
  return w5 ? dispatch_tc_xprop_fp8<BS, 0, 1>(p, maps, n_out, bf16, s) : dispatch_tc_xprop_fp8<BS, 0, 0>(p, maps, n_out, bf16, s);
}

// Arguments already checked by bsmm_xprop_fp8: axis 1, bsize 32 / 64, fp8 x and w, 16-bit y, aligned pointers, N > 0.
inline int tc_xprop_fp8(int x_dtype, int w_dtype, int y_dtype, int bsize, const int32_t* lut, int n_out, int n_in,
                        int blocks, const void* x, const void* w, void* y, int N, const float* x_scale_inv,
                        const float* w_scale_inv, cudaStream_t s) {
  if (!wgmma_device()) return fail(BSMM_E_NODEV, "bsmm_xprop_fp8: %s", err_buf());
  const uint64_t Cin = (uint64_t)n_in * bsize, Cout = (uint64_t)n_out * bsize;
  const CUtensorMapSwizzle swz = tmap_swizzle_for_row(bsize);
  XpropTmaps maps;
  if (int e = cached_tmap_2d(&maps.x, x_dtype, x, Cin, (uint64_t)N, Cin, bsize, 128, swz)) return e;
  const uint64_t w_rows = (uint64_t)(blocks > 0 ? blocks : 1) * bsize;     // no blocks: no LUT entry reads w
  if (int e = cached_tmap_2d(&maps.w, w_dtype, w, (uint64_t)bsize, w_rows, (uint64_t)bsize, bsize, bsize, swz)) return e;
  XpropFp8Params p;
  p.lut = lut; p.y = y; p.y_pitch = (long long)Cout; p.N = N;
  p.x_scale_inv = x_scale_inv; p.w_scale_inv = w_scale_inv;
  const bool bf = y_dtype == BSMM_BF16;
  return bsize == 32 ? dispatch_tc_xprop_fp8<32>(p, maps, n_out, x_dtype, w_dtype, bf, s)
                     : dispatch_tc_xprop_fp8<64>(p, maps, n_out, x_dtype, w_dtype, bf, s);
}

}  // namespace bsmm
