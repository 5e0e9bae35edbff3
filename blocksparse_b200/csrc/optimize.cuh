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

}  // namespace bsmm
