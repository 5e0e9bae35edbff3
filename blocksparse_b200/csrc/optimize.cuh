// Multi-tensor optimizer kernels (the reference's blocksparse/optimize.py): Adam with optional per-block gates and
// 16-bit moment codes, the global-norm reduction behind clip_by_global_norm, and the parameter EMA.
//
// Every launch covers up to MT_MAX tensors. Their table travels in the kernel parameters (__grid_constant__, so it is
// read from the constant bank and never copied to local memory), so a call makes no host-to-device copy and no host
// synchronisation. Each tensor is cut into chunks of MT_CHUNK elements; the grid has one CTA per chunk and a CTA finds
// its tensor by a binary search over the table's first-chunk indices. The partition depends on the list of sizes only.
#pragma once
#include <type_traits>
#include "common.cuh"

namespace bsmm {

constexpr int MT_MAX = 256;          // tensors per launch: 256 * 56 bytes of table stays under the 32,764-byte parameter limit
constexpr int MT_THREADS = 256;
constexpr int MT_CHUNK = 8192;       // elements per CTA: 8 vector steps of 4 elements per thread
// Elements per thread and vector step: 16 bytes of fp32, 8 of 16-bit data, so that each warp instruction covers one
// contiguous span. Eight elements per thread (16 bytes of 16-bit data, two 16-byte halves of fp32) made every fp32 access
// a half-sector stride and ran the fp32-moment Adam step at a third of the bandwidth on an H100 (DESIGN.md 7e).
constexpr int MT_VEC = 4;
constexpr int MT_NORM_THREADS = 1024;

struct MtTensor {
  const void* a;                     // adam: grad; norm: x; ema: param
  void* b;                           // adam: param; ema: average
  void* c;                           // adam: mean
  void* d;                           // adam: var
  const float* gate;                 // per-block gate or NULL
  long long size;                    // elements
  int chunk0;                        // first chunk of this tensor within the launch
  uint8_t dtype, codes, vec, bshift; // dtype of `a`; 16-bit moments; vector accesses; log2(bs*bs), 0 = ungated
};
static_assert(sizeof(MtTensor) == 56, "table entry layout");

struct MtTable {
  MtTensor t[MT_MAX];
  int n;
};

struct AdamConsts {
  const float* norm_scale;
  float lr, decay_mean, decay_var, epsilon, grad_scale, clip_sigma, saturate;
  int zero_infs, zero_nans;
};

__device__ __forceinline__ int mt_find(const MtTable& tab, int chunk) {
  int lo = 0, hi = tab.n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (tab.t[mid].chunk0 <= chunk) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// ---- the reference's 16-bit moment formats (ew_op_gpu.h:332-431) ------------------------------------------------------
// Mean: sign bit 15, exponent bits 14-9, mantissa bits 8-0: +-2^(e-60) (1 + f/512), code 0 = 0. Variance: exponent bits
// 15-10, mantissa bits 9-0: 2^(e-60) (1 + f/1024), code 0 = 0. The exponent bias to fp32 is 127 - 60 = 67.
__device__ __forceinline__ float mean_decode(uint16_t c) {
  if (c == 0) return 0.f;
  const uint32_t bits = ((uint32_t)(c & 0x8000) << 16) | ((((c >> 9) & 63u) + 67u) << 23) | ((uint32_t)(c & 511) << 14);
  return __uint_as_float(bits);
}
__device__ __forceinline__ float var_decode(uint16_t c) {
  if (c == 0) return 0.f;
  return __uint_as_float((((uint32_t)(c >> 10) + 67u) << 23) | ((uint32_t)(c & 1023) << 13));
}
// Clamp to the largest code (a NaN clamps to +max, as fminf / fmaxf order it), flush below the smallest non-zero code,
// else add half a code ulp to the magnitude and truncate: rounds half away from zero.
__device__ __forceinline__ uint16_t mean_encode(float v) {
  v = fmaxf(fminf(v, 15.984375f), -15.984375f);
  if (fabsf(v) < 8.690558038829121e-19f) return 0;              // 2^-60 (1 + 2^-9)
  const uint32_t u = __float_as_uint(v);
  const uint32_t mag = ((u & 0x7fffffffu) + (1u << 13)) >> 14;    // 8-bit exponent and 9-bit mantissa
  return (uint16_t)(((u >> 16) & 0x8000u) | (mag - (67u << 9)));
}
__device__ __forceinline__ uint16_t var_encode(float v) {
  v = fminf(v, 15.9921875f);
  if (!(v >= 8.682087709356578e-19f)) return 0;                  // 2^-60 (1 + 2^-10); v is finite here
  const uint32_t mag = (__float_as_uint(v) + (1u << 12)) >> 13;
  return (uint16_t)(mag - (67u << 10));
}

// ---- loads and stores of MT_VEC elements (vector) or 1 (scalar), converted to / from fp32 ---------------------------------
struct MeanCode {};
struct VarCode {};

template <typename T> struct Io;
template <> struct Io<float> {
  static __device__ __forceinline__ void ldv(const void* p, long long i, float* o) {
    const float4 a = *reinterpret_cast<const float4*>(static_cast<const float*>(p) + i);
    o[0] = a.x; o[1] = a.y; o[2] = a.z; o[3] = a.w;
  }
  static __device__ __forceinline__ void stv(void* p, long long i, const float* v) {
    *reinterpret_cast<float4*>(static_cast<float*>(p) + i) = make_float4(v[0], v[1], v[2], v[3]);
  }
  static __device__ __forceinline__ float ld1(const void* p, long long i) { return static_cast<const float*>(p)[i]; }
  static __device__ __forceinline__ void st1(void* p, long long i, float v) { static_cast<float*>(p)[i] = v; }
};
template <typename H> struct Io16 {                  // __half, __nv_bfloat16 and the two moment codes
  static __device__ __forceinline__ float dec(uint16_t c) {
    if constexpr (std::is_same<H, MeanCode>::value) return mean_decode(c);
    else if constexpr (std::is_same<H, VarCode>::value) return var_decode(c);
    else return to_f32<H>(*reinterpret_cast<const H*>(&c));
  }
  static __device__ __forceinline__ uint16_t enc(float v) {
    if constexpr (std::is_same<H, MeanCode>::value) return mean_encode(v);
    else if constexpr (std::is_same<H, VarCode>::value) return var_encode(v);
    else { const H h = from_f32<H>(v); return *reinterpret_cast<const uint16_t*>(&h); }
  }
  static __device__ __forceinline__ void ldv(const void* p, long long i, float* o) {
    const uint2 r = *reinterpret_cast<const uint2*>(static_cast<const uint16_t*>(p) + i);
    const uint32_t w[2] = {r.x, r.y};
#pragma unroll
    for (int j = 0; j < 2; ++j) { o[2 * j] = dec((uint16_t)(w[j] & 0xffff)); o[2 * j + 1] = dec((uint16_t)(w[j] >> 16)); }
  }
  static __device__ __forceinline__ void stv(void* p, long long i, const float* v) {
    uint32_t w[2];
#pragma unroll
    for (int j = 0; j < 2; ++j) w[j] = (uint32_t)enc(v[2 * j]) | ((uint32_t)enc(v[2 * j + 1]) << 16);
    *reinterpret_cast<uint2*>(static_cast<uint16_t*>(p) + i) = make_uint2(w[0], w[1]);
  }
  static __device__ __forceinline__ float ld1(const void* p, long long i) { return dec(static_cast<const uint16_t*>(p)[i]); }
  static __device__ __forceinline__ void st1(void* p, long long i, float v) { static_cast<uint16_t*>(p)[i] = enc(v); }
};
template <> struct Io<__half> : Io16<__half> {};
template <> struct Io<__nv_bfloat16> : Io16<__nv_bfloat16> {};
template <> struct Io<MeanCode> : Io16<MeanCode> {};
template <> struct Io<VarCode> : Io16<VarCode> {};

// zero_infs, then zero_nans, then the saturate clamp (optimize_op_gpu.cu:477-482)
__device__ __forceinline__ float mt_condition(float g, float saturate, int zero_infs, int zero_nans) {
  if (zero_infs && isinf(g)) g = 0.f;
  if (zero_nans && isnan(g)) g = 0.f;
  if (saturate != 0.f) g = fmaxf(fminf(g, saturate), -saturate);
  return g;
}

// Walks the elements [c0, c1) of one tensor: W = MT_VEC with vector accesses (c0 is a multiple of MT_VEC, so a vector
// group never straddles a gate block of bs*bs >= 64 elements), then the scalar tail; W = 1 throughout without them. Blocks whose
// gate is 0 are neither read nor written.
template <bool VEC, typename F>
__device__ __forceinline__ void mt_walk(const MtTensor& t, long long c0, long long c1, F&& body) {
  long long i = c0 + (long long)threadIdx.x * (VEC ? MT_VEC : 1);
  if (VEC) {
    const long long body_end = c0 + ((c1 - c0) & ~(long long)(MT_VEC - 1));
    for (; i < body_end; i += MT_THREADS * MT_VEC)
      if (!t.bshift || t.gate[i >> t.bshift] != 0.f) body(i, std::integral_constant<int, MT_VEC>());
    i = body_end + threadIdx.x;
  }
  for (; i < c1; i += MT_THREADS)
    if (!t.bshift || t.gate[i >> t.bshift] != 0.f) body(i, std::integral_constant<int, 1>());
}

template <typename T, int W>
__device__ __forceinline__ void mt_ld(const void* p, long long i, float* o) {
  if constexpr (W == MT_VEC) Io<T>::ldv(p, i, o); else o[0] = Io<T>::ld1(p, i);
}
template <typename T, int W>
__device__ __forceinline__ void mt_st(void* p, long long i, const float* v) {
  if constexpr (W == MT_VEC) Io<T>::stv(p, i, v); else Io<T>::st1(p, i, v[0]);
}

// ---- Adam ------------------------------------------------------------------------------------------------------------
template <typename TG, bool CODES, bool VEC>
__device__ __forceinline__ void adam_tensor(const MtTensor& t, long long c0, long long c1, const AdamConsts& k, float ns) {
  using TM = typename std::conditional<CODES, MeanCode, float>::type;
  using TV = typename std::conditional<CODES, VarCode, float>::type;
  const float scale = k.grad_scale * ns;
  mt_walk<VEC>(t, c0, c1, [&](long long i, auto w) {
    constexpr int W = decltype(w)::value;
    float g[W], p[W], m[W], v[W];
    mt_ld<TG, W>(t.a, i, g);
    mt_ld<float, W>(t.b, i, p);
    mt_ld<TM, W>(t.c, i, m);
    mt_ld<TV, W>(t.d, i, v);
#pragma unroll
    for (int j = 0; j < W; ++j) {
      float gj = mt_condition(g[j], k.saturate, k.zero_infs, k.zero_nans) * scale;
      v[j] = k.decay_var * v[j] + (1.f - k.decay_var) * gj * gj;
      const float sigma = sqrtf(v[j]);
      if (k.clip_sigma != 0.f) {
        const float clip = k.clip_sigma * sigma;
        gj = fminf(fmaxf(gj, -clip), clip);
      }
      m[j] = k.decay_mean * m[j] + (1.f - k.decay_mean) * gj;
      p[j] -= k.lr * m[j] / (sigma + k.epsilon);
    }
    mt_st<TM, W>(t.c, i, m);
    mt_st<TV, W>(t.d, i, v);
    mt_st<float, W>(t.b, i, p);
  });
}

template <typename TG, bool CODES>
__device__ __forceinline__ void adam_dispatch_vec(const MtTensor& t, long long c0, long long c1, const AdamConsts& k, float ns) {
  if (t.vec) adam_tensor<TG, CODES, true>(t, c0, c1, k, ns);
  else adam_tensor<TG, CODES, false>(t, c0, c1, k, ns);
}

__global__ void __launch_bounds__(MT_THREADS) mt_adam(const __grid_constant__ MtTable tab, const AdamConsts k) {
  const float ns = k.norm_scale ? *k.norm_scale : 1.f;
  if (ns == 0.f) return;                             // a non-finite global norm skips the step (optimize_op_gpu.cu:463-466)
  const MtTensor& t = tab.t[mt_find(tab, blockIdx.x)];
  const long long c0 = (long long)(blockIdx.x - t.chunk0) * MT_CHUNK;
  const long long c1 = min(c0 + MT_CHUNK, t.size);
  switch (t.dtype * 2 + t.codes) {
    case BSMM_F32 * 2:      adam_dispatch_vec<float, false>(t, c0, c1, k, ns); break;
    case BSMM_F32 * 2 + 1:  adam_dispatch_vec<float, true>(t, c0, c1, k, ns); break;
    case BSMM_F16 * 2:      adam_dispatch_vec<__half, false>(t, c0, c1, k, ns); break;
    case BSMM_F16 * 2 + 1:  adam_dispatch_vec<__half, true>(t, c0, c1, k, ns); break;
    case BSMM_BF16 * 2:     adam_dispatch_vec<__nv_bfloat16, false>(t, c0, c1, k, ns); break;
    default:                adam_dispatch_vec<__nv_bfloat16, true>(t, c0, c1, k, ns); break;
  }
}

// ---- EMA: ema -= (1 - decay) * (ema - param) -------------------------------------------------------------------------
template <typename TE, bool VEC>
__device__ __forceinline__ void ema_tensor(const MtTensor& t, long long c0, long long c1, float decay) {
  mt_walk<VEC>(t, c0, c1, [&](long long i, auto w) {
    constexpr int W = decltype(w)::value;
    float e[W], p[W];
    mt_ld<TE, W>(t.b, i, e);
    mt_ld<float, W>(t.a, i, p);
#pragma unroll
    for (int j = 0; j < W; ++j) e[j] -= (1.f - decay) * (e[j] - p[j]);
    mt_st<TE, W>(t.b, i, e);
  });
}

template <typename TE>
__global__ void __launch_bounds__(MT_THREADS) mt_ema(const __grid_constant__ MtTable tab, float decay) {
  const MtTensor& t = tab.t[mt_find(tab, blockIdx.x)];
  const long long c0 = (long long)(blockIdx.x - t.chunk0) * MT_CHUNK;
  const long long c1 = min(c0 + MT_CHUNK, t.size);
  if (t.vec) ema_tensor<TE, true>(t, c0, c1, decay);
  else ema_tensor<TE, false>(t, c0, c1, decay);
}

// ---- global norm: fp32 sum of squares per chunk, then one CTA adds the chunk sums in fp64 in index order -------------
struct NormConsts { float grad_scale, saturate; int zero_infs, zero_nans; };

template <typename TX, bool VEC>
__device__ __forceinline__ float sumsq_tensor(const MtTensor& t, long long c0, long long c1, const NormConsts& k) {
  float acc = 0.f;
  mt_walk<VEC>(t, c0, c1, [&](long long i, auto w) {
    constexpr int W = decltype(w)::value;
    float x[W];
    mt_ld<TX, W>(t.a, i, x);
#pragma unroll
    for (int j = 0; j < W; ++j) {
      const float y = mt_condition(x[j], k.saturate, k.zero_infs, k.zero_nans) * k.grad_scale;
      acc = fmaf(y, y, acc);
    }
  });
  return acc;
}

template <typename T, int THREADS>
__device__ __forceinline__ T block_sum_fixed(T v, T* red) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  if (threadIdx.x < 32) {
    v = threadIdx.x < THREADS / 32 ? red[threadIdx.x] : T(0);
#pragma unroll
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  }
  return v;                                          // valid in thread 0
}

template <typename TX>
__device__ __forceinline__ float sumsq_dispatch_vec(const MtTensor& t, long long c0, long long c1, const NormConsts& k) {
  return t.vec ? sumsq_tensor<TX, true>(t, c0, c1, k) : sumsq_tensor<TX, false>(t, c0, c1, k);
}

__global__ void __launch_bounds__(MT_THREADS) mt_sumsq(const __grid_constant__ MtTable tab, const NormConsts k, float* partial) {
  __shared__ float red[MT_THREADS / 32];
  const MtTensor& t = tab.t[mt_find(tab, blockIdx.x)];
  const long long c0 = (long long)(blockIdx.x - t.chunk0) * MT_CHUNK;
  const long long c1 = min(c0 + MT_CHUNK, t.size);
  float acc;
  switch (t.dtype) {
    case BSMM_F32: acc = sumsq_dispatch_vec<float>(t, c0, c1, k); break;
    case BSMM_F16: acc = sumsq_dispatch_vec<__half>(t, c0, c1, k); break;
    default:       acc = sumsq_dispatch_vec<__nv_bfloat16>(t, c0, c1, k); break;
  }
  acc = block_sum_fixed<float, MT_THREADS>(acc, red);
  if (threadIdx.x == 0) partial[blockIdx.x] = acc;
}

// norm = sqrt(sum); scale = clip_norm / max(norm, clip_norm) when norm is finite, else 0 (optimize_op_gpu.cu:1183-1232)
__global__ void __launch_bounds__(MT_NORM_THREADS) mt_norm_finish(const float* partial, int chunks, float clip_norm,
                                                                   float* norm, float* scale) {
  __shared__ double red[MT_NORM_THREADS / 32];
  double acc = 0.0;
  for (int i = threadIdx.x; i < chunks; i += MT_NORM_THREADS) acc += (double)partial[i];
  acc = block_sum_fixed<double, MT_NORM_THREADS>(acc, red);
  if (threadIdx.x == 0) {
    const float n = (float)sqrt(acc);
    *norm = n;
    *scale = isfinite(n) ? clip_norm / fmaxf(n, clip_norm) : 0.f;
  }
}

// ---- host side: table building and launches --------------------------------------------------------------------------
inline long long mt_chunks(long long size) { return (size + MT_CHUNK - 1) / MT_CHUNK; }

// Splits the non-empty tensors into launches of at most MT_MAX tensors and 2^31 - 1 chunks; fill(i, entry) sets the
// pointers and flags of tensor i, launch(table, chunks, first chunk of the call) enqueues one kernel.
template <typename Fill, typename Launch>
inline int mt_for_launches(int n, const long long* sizes, Fill&& fill, Launch&& launch) {
  MtTable tab;
  tab.n = 0;
  long long chunks = 0, base = 0;
  for (int i = 0; i <= n; ++i) {
    const long long c = i < n ? mt_chunks(sizes[i]) : 0;
    if (tab.n && (i == n || tab.n == MT_MAX || chunks + c > 0x7fffffffLL)) {
      if (int e = launch(tab, (int)chunks, base)) return e;
      base += chunks;
      tab.n = 0;
      chunks = 0;
    }
    if (i == n || c == 0) continue;
    MtTensor& t = tab.t[tab.n++];
    t = MtTensor{};
    t.size = sizes[i];
    t.chunk0 = (int)chunks;
    fill(i, t);
    chunks += c;
  }
  return 0;
}

// ---- Adafactor (the reference's optimize_op_gpu.cu:8-365) -------------------------------------------------------------
// A (C, K) param with C > 1 keeps rv[C] and cv[K] (factored); any other keeps cv per element. One step is five launches per
// table of tensors:
//   1. mt_adafactor_stats   per tile of a factored grad: the tile's row and column sums of g^2 + eps into the workspace;
//                           per chunk of an unfactored one: cv updated in place and the chunk's sum of x^2
//   2. mt_adafactor_finish  per entry of rv / cv: its partials added in fp64 in tile order, then the decayed update
//   3. mt_adafactor_sumsq   per tile of a factored grad: the sum of g^2 / (rv[c] cv[k]), read again from the grad
//   4. mt_adafactor_rate    per tensor: mean(rv), rms = mean(rv) mean(g^2 / (rv cv)) (or mean(x^2)), the update rate
//   5. mt_adafactor_apply   per tile: the grad read a third time, x formed again, p -= rate x
// x is never stored: the workspace holds partial sums and two scalars per tensor. Every sum has a fixed partition and
// order (no atomics), so two calls give the same bits. A factored tile is AF_TR rows by AF_TK columns; warp w takes rows
// w, w + 8, ... and each lane 4 columns of them, so a lane keeps its column sums (and 1 / sqrt(cv)) in registers.
constexpr int AF_MAX = 384;          // tensors per launch: 384 * 72 bytes of table + AfConsts stay under 32,764 bytes
constexpr int AF_THREADS = 256;
constexpr int AF_WARPS = AF_THREADS / 32;
constexpr int AF_TR = 64;
constexpr int AF_TK = 128;
constexpr int AF_CHUNK = AF_TR * AF_TK;       // elements per CTA of an unfactored tensor
constexpr int AF_FIN = 256;                   // rv / cv entries per CTA of the finish pass

struct AfTensor {
  const void* g;
  float* p;
  float* cv;
  float* rv;                         // NULL: unfactored
  long long rows, cols;              // factored: C > 1 and K; unfactored: 1 and the size
  long long ws;                      // first workspace float of this tensor
  int tile0;                         // first tile (passes 1, 3 and 5) of this tensor within the launch
  int fin0;                          // first CTA of the finish pass (factored tensors only)
  uint8_t dtype, vec, pad[6];        // dtype of g; 16-byte accesses (every pointer aligned and K % 4 == 0)
};
static_assert(sizeof(AfTensor) == 72, "table entry layout");

struct AfTable {
  AfTensor t[AF_MAX];
  int n;
};

struct AfConsts {
  const float* norm_scale;
  float* ws;
  float lr, decay, epsilon, grad_scale, clip_thresh, saturate;
  int zero_infs, zero_nans;
};
static_assert(sizeof(AfTable) + sizeof(AfConsts) <= 32764, "the table must fit the kernel parameters");

// Workspace floats of a tensor, from its first: [0] mean(rv), [1] update rate, then one sum of squares per tile, then
// (factored) the row partials [tile column][C] and the column partials [tile row][K].
__host__ __device__ inline long long af_tile_rows(long long C) { return (C + AF_TR - 1) / AF_TR; }
__host__ __device__ inline long long af_tile_cols(long long K) { return (K + AF_TK - 1) / AF_TK; }
__host__ __device__ inline long long af_tiles(long long rows, long long cols) {
  return rows > 1 ? af_tile_rows(rows) * af_tile_cols(cols) : (cols + AF_CHUNK - 1) / AF_CHUNK;
}
__host__ __device__ inline long long af_ws_floats(long long rows, long long cols) {
  if (rows * cols == 0) return 0;
  const long long tiles = af_tiles(rows, cols);
  return 2 + tiles + (rows > 1 ? rows * af_tile_cols(cols) + af_tile_rows(rows) * cols : 0);
}

__device__ __forceinline__ int af_find_tile(const AfTable& tab, int b) {
  int lo = 0, hi = tab.n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (tab.t[mid].tile0 <= b) lo = mid; else hi = mid - 1;
  }
  return lo;
}
// Unfactored tensors have no finish CTAs and share fin0 with the next tensor: the last tensor at or below b owns b.
__device__ __forceinline__ int af_find_fin(const AfTable& tab, int b) {
  int lo = 0, hi = tab.n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (tab.t[mid].fin0 <= b) lo = mid; else hi = mid - 1;
  }
  return lo;
}

__device__ __forceinline__ float af_norm_scale(const AfConsts& k) { return k.norm_scale ? *k.norm_scale : 1.f; }

// Column of a lane's j-th element in a factored tile: 4 adjacent ones with 16-byte accesses, a stride of 32 without.
template <bool VEC>
__device__ __forceinline__ long long af_col(long long k0, int lane, int j) { return VEC ? k0 + 4 * lane + j : k0 + lane + 32 * j; }

// The 4 elements of row `row` a lane owns (0 past the last column), converted to fp32.
template <typename T, bool VEC>
__device__ __forceinline__ void af_ld_row(const void* p, long long row, long long K, long long k0, int lane, float* v) {
  if constexpr (VEC) {
    if (af_col<true>(k0, lane, 0) < K) { Io<T>::ldv(p, row * K + af_col<true>(k0, lane, 0), v); return; }
#pragma unroll
    for (int j = 0; j < 4; ++j) v[j] = 0.f;
  } else {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const long long c = af_col<false>(k0, lane, j);
      v[j] = c < K ? Io<T>::ld1(p, row * K + c) : 0.f;
    }
  }
}

template <bool VEC>
__device__ __forceinline__ void af_st_row(float* p, long long row, long long K, long long k0, int lane, const float* v) {
  if constexpr (VEC) {
    if (af_col<true>(k0, lane, 0) < K) Io<float>::stv(p, row * K + af_col<true>(k0, lane, 0), v);
  } else {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const long long c = af_col<false>(k0, lane, j);
      if (c < K) p[row * K + c] = v[j];
    }
  }
}

// Elements [c0, c1) of an unfactored chunk: MT_VEC at a time with 16-byte accesses, then the scalar tail.
template <bool VEC, typename F>
__device__ __forceinline__ void af_walk(long long c0, long long c1, F&& body) {
  long long i = c0 + (long long)threadIdx.x * (VEC ? MT_VEC : 1);
  if (VEC) {
    const long long body_end = c0 + ((c1 - c0) & ~(long long)(MT_VEC - 1));
    for (; i < body_end; i += AF_THREADS * MT_VEC) body(i, std::integral_constant<int, MT_VEC>());
    i = body_end + threadIdx.x;
  }
  for (; i < c1; i += AF_THREADS) body(i, std::integral_constant<int, 1>());
}

// pass 1
template <typename TG, bool VEC>
__device__ __forceinline__ void af_stats(const AfTensor& t, long long tile, const AfConsts& k, float scale, float* red) {
  float* ws = k.ws + t.ws;
  if (!t.rv) {
    const long long c0 = tile * AF_CHUNK, c1 = min(c0 + AF_CHUNK, t.cols);
    float acc = 0.f;
    af_walk<VEC>(c0, c1, [&](long long i, auto w) {
      constexpr int W = decltype(w)::value;
      float g[W], v[W];
      mt_ld<TG, W>(t.g, i, g);
      mt_ld<float, W>(t.cv, i, v);
#pragma unroll
      for (int j = 0; j < W; ++j) {
        const float gj = mt_condition(g[j], k.saturate, k.zero_infs, k.zero_nans) * scale;
        v[j] = k.decay * v[j] + (1.f - k.decay) * (gj * gj + k.epsilon);
        const float x = gj * rsqrtf(v[j]);
        acc = fmaf(x, x, acc);
      }
      mt_st<float, W>(t.cv, i, v);
    });
    acc = block_sum_fixed<float, AF_THREADS>(acc, red);
    if (threadIdx.x == 0) ws[2 + tile] = acc;
    return;
  }
  const long long C = t.rows, K = t.cols, ntc = af_tile_cols(K);
  const long long tr = tile / ntc, tc = tile - tr * ntc;
  const long long r0 = tr * AF_TR, r1 = min(r0 + AF_TR, C), k0 = tc * AF_TK;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float* rowpart = ws + 2 + af_tiles(C, K) + tc * C;
  float* colpart = ws + 2 + af_tiles(C, K) + C * ntc + tr * K;
  float col[4] = {0.f, 0.f, 0.f, 0.f};
  for (long long r = r0 + warp; r < r1; r += AF_WARPS) {
    float g[4];
    af_ld_row<TG, VEC>(t.g, r, K, k0, lane, g);
    float rs = 0.f;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float gj = mt_condition(g[j], k.saturate, k.zero_infs, k.zero_nans) * scale;
      const float s = af_col<VEC>(k0, lane, j) < K ? gj * gj + k.epsilon : 0.f;
      col[j] += s;
      rs += s;
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) rs += __shfl_xor_sync(0xffffffffu, rs, o);
    if (lane == 0) rowpart[r] = rs;
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) red[warp * AF_TK + (int)(af_col<VEC>(0, lane, j))] = col[j];
  __syncthreads();
  if (threadIdx.x < AF_TK && k0 + threadIdx.x < K) {
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < AF_WARPS; ++w) s += red[w * AF_TK + threadIdx.x];
    colpart[k0 + threadIdx.x] = s;
  }
}

template <typename TG>
__device__ __forceinline__ void af_stats_vec(const AfTensor& t, long long tile, const AfConsts& k, float scale, float* red) {
  if (t.vec) af_stats<TG, true>(t, tile, k, scale, red); else af_stats<TG, false>(t, tile, k, scale, red);
}

__global__ void __launch_bounds__(AF_THREADS) mt_adafactor_stats(const __grid_constant__ AfTable tab, const AfConsts k) {
  __shared__ float red[AF_WARPS * AF_TK];
  const float ns = af_norm_scale(k);
  if (ns == 0.f) return;                             // a non-finite global norm skips the step
  const AfTensor& t = tab.t[af_find_tile(tab, blockIdx.x)];
  const long long tile = blockIdx.x - t.tile0;
  const float scale = k.grad_scale * ns;
  switch (t.dtype) {
    case BSMM_F32: af_stats_vec<float>(t, tile, k, scale, red); break;
    case BSMM_F16: af_stats_vec<__half>(t, tile, k, scale, red); break;
    default:       af_stats_vec<__nv_bfloat16>(t, tile, k, scale, red); break;
  }
}

// pass 2: rv[c] = decay rv[c] + (1 - decay) (row sum) / K, cv[k] = decay cv[k] + (1 - decay) (column sum) / C
__global__ void __launch_bounds__(AF_FIN) mt_adafactor_finish(const __grid_constant__ AfTable tab, const AfConsts k) {
  if (af_norm_scale(k) == 0.f) return;
  const AfTensor& t = tab.t[af_find_fin(tab, blockIdx.x)];
  const long long C = t.rows, K = t.cols, ntc = af_tile_cols(K), ntr = af_tile_rows(C);
  const long long e = (long long)(blockIdx.x - t.fin0) * AF_FIN + threadIdx.x;
  const float* part = k.ws + t.ws + 2 + af_tiles(C, K);
  if (e < C) {
    double s = 0.0;
    for (long long j = 0; j < ntc; ++j) s += (double)part[j * C + e];
    t.rv[e] = k.decay * t.rv[e] + (1.f - k.decay) * (float)(s / (double)K);
  } else if (e < C + K) {
    const long long c = e - C;
    part += C * ntc;
    double s = 0.0;
    for (long long i = 0; i < ntr; ++i) s += (double)part[i * K + c];
    t.cv[c] = k.decay * t.cv[c] + (1.f - k.decay) * (float)(s / (double)C);
  }
}

// pass 3: sum of (g / sqrt(rv[c] cv[k]))^2 over a factored tile
template <typename TG, bool VEC>
__device__ __forceinline__ float af_sumsq(const AfTensor& t, long long tile, const AfConsts& k, float scale) {
  const long long C = t.rows, K = t.cols, ntc = af_tile_cols(K);
  const long long tr = tile / ntc, tc = tile - tr * ntc;
  const long long r0 = tr * AF_TR, r1 = min(r0 + AF_TR, C), k0 = tc * AF_TK;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float rc[4];
  af_ld_row<float, VEC>(t.cv, 0, K, k0, lane, rc);
#pragma unroll
  for (int j = 0; j < 4; ++j) rc[j] = af_col<VEC>(k0, lane, j) < K ? rsqrtf(rc[j]) : 0.f;
  float acc = 0.f;
  for (long long r = r0 + warp; r < r1; r += AF_WARPS) {
    float g[4];
    af_ld_row<TG, VEC>(t.g, r, K, k0, lane, g);
    const float rr = rsqrtf(t.rv[r]);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float y = mt_condition(g[j], k.saturate, k.zero_infs, k.zero_nans) * scale * rr * rc[j];
      acc = fmaf(y, y, acc);
    }
  }
  return acc;
}

__global__ void __launch_bounds__(AF_THREADS) mt_adafactor_sumsq(const __grid_constant__ AfTable tab, const AfConsts k) {
  __shared__ float red[AF_WARPS];
  const float ns = af_norm_scale(k);
  if (ns == 0.f) return;
  const AfTensor& t = tab.t[af_find_tile(tab, blockIdx.x)];
  if (!t.rv) return;                                 // unfactored: pass 1 wrote the partials
  const long long tile = blockIdx.x - t.tile0;
  const float scale = k.grad_scale * ns;
  float acc;
  switch (t.dtype * 2 + t.vec) {
    case BSMM_F32 * 2:      acc = af_sumsq<float, false>(t, tile, k, scale); break;
    case BSMM_F32 * 2 + 1:  acc = af_sumsq<float, true>(t, tile, k, scale); break;
    case BSMM_F16 * 2:      acc = af_sumsq<__half, false>(t, tile, k, scale); break;
    case BSMM_F16 * 2 + 1:  acc = af_sumsq<__half, true>(t, tile, k, scale); break;
    case BSMM_BF16 * 2:     acc = af_sumsq<__nv_bfloat16, false>(t, tile, k, scale); break;
    default:                acc = af_sumsq<__nv_bfloat16, true>(t, tile, k, scale); break;
  }
  acc = block_sum_fixed<float, AF_THREADS>(acc, red);
  if (threadIdx.x == 0) k.ws[t.ws + 2 + tile] = acc;
}

// pass 4: one CTA per tensor. rate = lr / max(1, sqrt(rms) / clip_thresh), rms = mean(x^2).
__global__ void __launch_bounds__(AF_THREADS) mt_adafactor_rate(const __grid_constant__ AfTable tab, const AfConsts k) {
  __shared__ double red[AF_WARPS];
  if (af_norm_scale(k) == 0.f) return;
  const AfTensor& t = tab.t[blockIdx.x];
  float* ws = k.ws + t.ws;
  const long long tiles = af_tiles(t.rows, t.cols);
  double sq = 0.0, rvs = 0.0;
  for (long long i = threadIdx.x; i < tiles; i += AF_THREADS) sq += (double)ws[2 + i];
  sq = block_sum_fixed<double, AF_THREADS>(sq, red);
  __syncthreads();                                   // red is reused
  if (t.rv) {
    for (long long i = threadIdx.x; i < t.rows; i += AF_THREADS) rvs += (double)t.rv[i];
    rvs = block_sum_fixed<double, AF_THREADS>(rvs, red);
  }
  if (threadIdx.x == 0) {
    const double n = (double)t.rows * (double)t.cols;
    const float rv_mean = t.rv ? (float)(rvs / (double)t.rows) : 1.f;
    const double rms = t.rv ? (double)rv_mean * sq / n : sq / n;
    ws[0] = rv_mean;
    ws[1] = (float)((double)k.lr / fmax(1.0, sqrt(rms) / (double)k.clip_thresh));
  }
}

// pass 5: p -= rate * x, x = g / sqrt(rv[c] / mean(rv)) / sqrt(cv[k]) or g / sqrt(cv)
template <typename TG, bool VEC>
__device__ __forceinline__ void af_apply(const AfTensor& t, long long tile, const AfConsts& k, float scale) {
  const float* ws = k.ws + t.ws;
  const float rate = ws[1];
  if (!t.rv) {
    const long long c0 = tile * AF_CHUNK, c1 = min(c0 + AF_CHUNK, t.cols);
    af_walk<VEC>(c0, c1, [&](long long i, auto w) {
      constexpr int W = decltype(w)::value;
      float g[W], v[W], p[W];
      mt_ld<TG, W>(t.g, i, g);
      mt_ld<float, W>(t.cv, i, v);
      mt_ld<float, W>(t.p, i, p);
#pragma unroll
      for (int j = 0; j < W; ++j) {
        const float gj = mt_condition(g[j], k.saturate, k.zero_infs, k.zero_nans) * scale;
        p[j] -= rate * (gj * rsqrtf(v[j]));
      }
      mt_st<float, W>(t.p, i, p);
    });
    return;
  }
  const float rv_mean = ws[0];
  const long long C = t.rows, K = t.cols, ntc = af_tile_cols(K);
  const long long tr = tile / ntc, tc = tile - tr * ntc;
  const long long r0 = tr * AF_TR, r1 = min(r0 + AF_TR, C), k0 = tc * AF_TK;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float rc[4];
  af_ld_row<float, VEC>(t.cv, 0, K, k0, lane, rc);
#pragma unroll
  for (int j = 0; j < 4; ++j) rc[j] = af_col<VEC>(k0, lane, j) < K ? rsqrtf(rc[j]) : 0.f;
  for (long long r = r0 + warp; r < r1; r += AF_WARPS) {
    float g[4], p[4];
    af_ld_row<TG, VEC>(t.g, r, K, k0, lane, g);
    af_ld_row<float, VEC>(t.p, r, K, k0, lane, p);
    const float rr = rsqrtf(t.rv[r] / rv_mean);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float gj = mt_condition(g[j], k.saturate, k.zero_infs, k.zero_nans) * scale;
      p[j] -= rate * (gj * rr * rc[j]);
    }
    af_st_row<VEC>(t.p, r, K, k0, lane, p);
  }
}

__global__ void __launch_bounds__(AF_THREADS) mt_adafactor_apply(const __grid_constant__ AfTable tab, const AfConsts k) {
  const float ns = af_norm_scale(k);
  if (ns == 0.f) return;
  const AfTensor& t = tab.t[af_find_tile(tab, blockIdx.x)];
  const long long tile = blockIdx.x - t.tile0;
  const float scale = k.grad_scale * ns;
  switch (t.dtype * 2 + t.vec) {
    case BSMM_F32 * 2:      af_apply<float, false>(t, tile, k, scale); break;
    case BSMM_F32 * 2 + 1:  af_apply<float, true>(t, tile, k, scale); break;
    case BSMM_F16 * 2:      af_apply<__half, false>(t, tile, k, scale); break;
    case BSMM_F16 * 2 + 1:  af_apply<__half, true>(t, tile, k, scale); break;
    case BSMM_BF16 * 2:     af_apply<__nv_bfloat16, false>(t, tile, k, scale); break;
    default:                af_apply<__nv_bfloat16, true>(t, tile, k, scale); break;
  }
}

// Splits the non-empty tensors into tables of at most AF_MAX tensors, 2^31 - 1 tiles and 2^31 - 1 finish CTAs;
// fill(i, entry) sets the pointers and flags of tensor i, launch(table, tiles, finish CTAs) enqueues the five passes.
template <typename Fill, typename Launch>
inline int af_for_launches(int n, const long long* rows, const long long* cols, Fill&& fill, Launch&& launch) {
  AfTable tab;
  tab.n = 0;
  long long tiles = 0, fins = 0, ws = 0;
  for (int i = 0; i <= n; ++i) {
    const bool live = i < n && rows[i] * cols[i] > 0;
    const long long c = live ? af_tiles(rows[i], cols[i]) : 0;
    const long long f = live && rows[i] > 1 ? (rows[i] + cols[i] + AF_FIN - 1) / AF_FIN : 0;
    if (tab.n && (i == n || tab.n == AF_MAX || tiles + c > 0x7fffffffLL || fins + f > 0x7fffffffLL)) {
      if (int e = launch(tab, (int)tiles, (int)fins)) return e;
      tab.n = 0;
      tiles = fins = 0;
    }
    if (!live) continue;
    AfTensor& t = tab.t[tab.n++];
    t = AfTensor{};
    t.rows = rows[i];
    t.cols = cols[i];
    t.ws = ws;
    t.tile0 = (int)tiles;
    t.fin0 = (int)fins;
    fill(i, t);
    tiles += c;
    fins += f;
    ws += af_ws_floats(rows[i], cols[i]);
  }
  return 0;
}

}  // namespace bsmm
