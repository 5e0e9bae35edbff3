// Quantization to narrow float formats and its statistics (bsmm_quantize, bsmm_quantize_stats in include/bsmm_b200.h).
//
// A format is (ebits, fbits, denorm) plus an exponent exp_max that lives in device memory, one int64 record per tensor.
// Every kernel derives the format's constants from that record on the device (q_format), so the host never reads it:
//   em        = clamp(exp_max + 127, top, 254), top = 2^ebits - 1 (254 for ebits 8, whose top bin is inf in fp32)
//   exp_min   = max(em - top + 1 - (denorm ? fbits : 0), 2)
//   max_float = bits ((em << 23) | 0x7fffff) & mask, mask = ~0 << (23 - fbits);  min_float = bits exp_min << 23
//   ftz_float = bits ((exp_min - 1) << 23) | 0x400000;                            exp_norm = (exp_min - 1 - (denorm ? 0 : fbits)) << 23
// The upper clamp at 254 keeps max_float finite whatever the record holds.
//
// One element (q_round): NaN stays NaN (0x7fffffff). Otherwise add r * 2^E with E the element's exponent, rounding
// toward zero and flushing fp32 subnormals (fma.rz.ftz), and clear the bits below fbits: r = 2^-(fbits+1) rounds half an
// ulp away from zero; stochastic rounding takes r = fp32(u) 2^-(fbits+32) for a 32-bit random word u, a uniform fraction
// of one ulp. Then clamp to +-max_float, give +0 below min_float, and round the format's subnormal range by moving
// exp_min to fp32's smallest normal exponent (- exp_norm), multiplying by 2^-23 (round to nearest even in fp32's
// subnormals), multiplying back by 2^23 and moving back (+ exp_norm). This is the reference kernel's arithmetic step for
// step (quantize_op_gpu.cu), so results agree with it bit for bit on every non-NaN input.
//
// Random words come from the Philox4x32-10 state of dropout ([seed, call], int64, on the device): element e of the
// tensor at position i of a call takes word e % 4 at counter (e / 4, call + i), and a one-thread kernel then advances
// call by the number of tensors, so results depend on (seed, call, x) only.
//
// Statistics (q_stats + q_stats_finish): one CTA per chunk of Q_CHUNK elements adds |x| and x^2 in fp64 per thread and
// counts saturated and flushed elements in integers; the warps are combined in a fixed order and each chunk writes one
// QPart. One CTA per tensor then adds its chunks' parts in fp64 in chunk order. Nothing depends on timing, so two calls
// give the same bits. In quantize mode the thresholds come from the record and the finish pass writes the next exponent
// back into it, on the same stream before the quantize launch reads it.
#pragma once
#include "ewops.cuh"

namespace bsmm {

constexpr int Q_MAX = 256;           // tensors per launch: 256 * 48 bytes of table
constexpr int Q_THREADS = 256;
constexpr int Q_CHUNK = 8192;        // elements per CTA
constexpr int Q_STATS = 5;           // mean |x|, stdv, sat %, ftz %, max |x| (the reference's QuantStats order)

struct QTensor {
  const void* x;
  void* y;                           // quantize only
  long long* exp;                    // exponent record; NULL in log mode of the statistics
  long long size;
  long long index;                   // position in the caller's list: Philox call offset and statistics row
  int chunk0;                        // first chunk of this tensor within the launch
  uint8_t vec;                       // 16-byte accesses
};
static_assert(sizeof(QTensor) == 48, "table entry layout");

struct QTable {
  QTensor t[Q_MAX];
  int n;
};

struct QConsts {
  const long long* entropy;          // stochastic only
  int ebits, fbits, denorm, stoch;
};

struct QStatConsts {
  float* stats;                      // [n][Q_STATS]
  void* parts;                       // QPart per chunk
  float sat_val, ftz_val, stdv_mul;  // thresholds of log mode
  int ebits, fbits, denorm, mode, bias_pad, half;
};

struct QPart {
  double sabs, ssq;
  unsigned long long sat, ftz;
  float vmax;
};

struct QFormat {
  float max_float, min_float, ftz_float;
  unsigned exp_norm;
};

__host__ __device__ __forceinline__ int q_top(int ebits) { return ebits == 8 ? 254 : (1 << ebits) - 1; }

// biased exponent em of a record value, clamped so that max_float stays finite
__device__ __forceinline__ int q_biased(long long e, int ebits) {
  const long long top = q_top(ebits);
  e = e > 1000 ? 1000 : e < -1000 ? -1000 : e;
  const long long b = e + 127;
  return (int)(b < top ? top : b > 254 ? 254 : b);
}

__device__ __forceinline__ QFormat q_format(long long e, int ebits, int fbits, int denorm) {
  const int em = q_biased(e, ebits);
  int exp_min = em - q_top(ebits) + 1 - (denorm ? fbits : 0);
  if (exp_min < 2) exp_min = 2;
  const unsigned mask = 0xffffffffu << (23 - fbits);
  QFormat f;
  f.max_float = __uint_as_float((((unsigned)em << 23) | 0x7fffffu) & mask);
  f.min_float = __uint_as_float((unsigned)exp_min << 23);
  f.ftz_float = __uint_as_float(((unsigned)(exp_min - 1) << 23) | 0x400000u);
  f.exp_norm = (unsigned)(exp_min - 1 - (denorm ? 0 : fbits)) << 23;      // wraps as the reference's does
  return f;
}

__device__ __forceinline__ float q_round(float x, float r, unsigned mask, const QFormat& f) {
  if (isnan(x)) return __uint_as_float(0x7fffffffu);
  const float se = __uint_as_float(__float_as_uint(x) & 0xff800000u);
  float v;
  asm("fma.rz.ftz.f32 %0, %1, %2, %3;" : "=f"(v) : "f"(se), "f"(r), "f"(x));
  v = __uint_as_float(__float_as_uint(v) & mask);
  v = fminf(fmaxf(v, -f.max_float), f.max_float);
  if (fabsf(v) < f.min_float) return 0.f;
  const float s = __fmul_rz(__fmul_rn(__uint_as_float(__float_as_uint(v) - f.exp_norm), 0x1p-23f), 0x1p23f);
  return __uint_as_float(__float_as_uint(s) + f.exp_norm);
}

// ---- element access: V elements at e (16 bytes) or 1 ----------------------------------------------------------------
template <typename T> struct QIo;
template <> struct QIo<float> {
  static constexpr int V = 4;
  static __device__ __forceinline__ void ldv(const void* p, long long e, float* o) {
    const float4 a = *reinterpret_cast<const float4*>(static_cast<const float*>(p) + e);
    o[0] = a.x; o[1] = a.y; o[2] = a.z; o[3] = a.w;
  }
  static __device__ __forceinline__ void stv(void* p, long long e, const float* v) {
    *reinterpret_cast<float4*>(static_cast<float*>(p) + e) = make_float4(v[0], v[1], v[2], v[3]);
  }
  static __device__ __forceinline__ float ld1(const void* p, long long e) { return static_cast<const float*>(p)[e]; }
  static __device__ __forceinline__ void st1(void* p, long long e, float v) { static_cast<float*>(p)[e] = v; }
};
// bf16 / fp16 as raw 16-bit words. A quantized value with fbits <= 7 has no bit set below bit 16 of its fp32 pattern
// (tests/test_quantize_oracle.py checks this over every format), so the bf16 store keeps the top half as it is.
template <typename H> struct QIo16 {
  static constexpr int V = 8;
  static __device__ __forceinline__ float dec(unsigned c) {
    if constexpr (std::is_same<H, __half>::value) return __half2float(__ushort_as_half((unsigned short)c));
    else return __uint_as_float(c << 16);
  }
  static __device__ __forceinline__ unsigned enc(float v) { return __float_as_uint(v) >> 16; }
  static __device__ __forceinline__ void ldv(const void* p, long long e, float* o) {
    const uint4 r = *reinterpret_cast<const uint4*>(static_cast<const uint16_t*>(p) + e);
    const unsigned w[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) { o[2 * j] = dec(w[j] & 0xffffu); o[2 * j + 1] = dec(w[j] >> 16); }
  }
  static __device__ __forceinline__ void stv(void* p, long long e, const float* v) {
    unsigned w[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) w[j] = enc(v[2 * j]) | (enc(v[2 * j + 1]) << 16);
    *reinterpret_cast<uint4*>(static_cast<uint16_t*>(p) + e) = make_uint4(w[0], w[1], w[2], w[3]);
  }
  static __device__ __forceinline__ float ld1(const void* p, long long e) { return dec(static_cast<const uint16_t*>(p)[e]); }
  static __device__ __forceinline__ void st1(void* p, long long e, float v) {
    static_cast<uint16_t*>(p)[e] = (uint16_t)enc(v);
  }
};
template <> struct QIo<__nv_bfloat16> : QIo16<__nv_bfloat16> {};
template <> struct QIo<__half> : QIo16<__half> {};

__device__ __forceinline__ int q_find(const QTable& tab, int chunk) {
  int lo = 0, hi = tab.n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (tab.t[mid].chunk0 <= chunk) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// Calls body(e, width) over the elements [c0, c1) of a chunk: V at a time with 16-byte accesses, then one at a time.
template <int V, bool VEC, typename F>
__device__ __forceinline__ void q_walk(long long c0, long long c1, F&& body) {
  long long e = c0;
  if constexpr (VEC) {
    const long long end = c0 + ((c1 - c0) / V) * V;
#pragma unroll 4
    for (e = c0 + (long long)threadIdx.x * V; e < end; e += (long long)Q_THREADS * V)
      body(e, std::integral_constant<int, V>());
    e = end;
  }
  for (e += threadIdx.x; e < c1; e += Q_THREADS) body(e, std::integral_constant<int, 1>());
}

// ---- quantize --------------------------------------------------------------------------------------------------------
template <typename T, bool VEC, bool STOCH>
__device__ __forceinline__ void q_tensor(const QTensor& t, long long c0, long long c1, const QConsts& k) {
  const QFormat f = q_format(*t.exp, k.ebits, k.fbits, k.denorm);
  const unsigned mask = 0xffffffffu << (23 - k.fbits);
  uint2 key = make_uint2(0, 0);
  unsigned long long call = 0;
  if constexpr (STOCH) {
    const unsigned long long seed = (unsigned long long)k.entropy[0];
    key = make_uint2((unsigned)seed, (unsigned)(seed >> 32));
    call = (unsigned long long)k.entropy[1] + (unsigned long long)t.index;
  }
  const float r0 = __uint_as_float((unsigned)((STOCH ? 95 : 126) - k.fbits) << 23);
  q_walk<QIo<T>::V, VEC>(c0, c1, [&](long long e, auto w) {
    constexpr int W = decltype(w)::value;
    float v[W];
    if constexpr (W == 1) v[0] = QIo<T>::ld1(t.x, e); else QIo<T>::ldv(t.x, e, v);
    unsigned u[W > 4 ? W : 4];
    if constexpr (STOCH) {
#pragma unroll
      for (int g = 0; g < (W + 3) / 4; ++g) {
        const unsigned long long blk = (unsigned long long)(e / 4 + g);
        const uint4 p = philox4x32_10(make_uint4((unsigned)blk, (unsigned)(blk >> 32), (unsigned)call,
                                                 (unsigned)(call >> 32)), key);
        u[4 * g] = p.x; u[4 * g + 1] = p.y; u[4 * g + 2] = p.z; u[4 * g + 3] = p.w;
      }
      if constexpr (W == 1) u[0] = u[e & 3];
    }
#pragma unroll
    for (int j = 0; j < W; ++j) v[j] = q_round(v[j], STOCH ? __fmul_rn(r0, __uint2float_rn(u[j])) : r0, mask, f);
    if constexpr (W == 1) QIo<T>::st1(t.y, e, v[0]); else QIo<T>::stv(t.y, e, v);
  });
}

template <typename T, bool STOCH>
__global__ void __launch_bounds__(Q_THREADS) q_quantize(const __grid_constant__ QTable tab, const QConsts k) {
  const QTensor& t = tab.t[q_find(tab, blockIdx.x)];
  const long long c0 = (long long)(blockIdx.x - t.chunk0) * Q_CHUNK;
  const long long c1 = min(c0 + Q_CHUNK, t.size);
  if (t.vec) q_tensor<T, true, STOCH>(t, c0, c1, k);
  else q_tensor<T, false, STOCH>(t, c0, c1, k);
}

__global__ void q_advance(long long* state, long long by) { state[1] += by; }

// ---- statistics ------------------------------------------------------------------------------------------------------
template <typename T, bool VEC>
__device__ __forceinline__ QPart q_stats_tensor(const QTensor& t, long long c0, long long c1, float satv, float ftzv,
                                                bool half) {
  QPart p = {0.0, 0.0, 0ull, 0ull, 0.f};
  q_walk<QIo<T>::V, VEC>(c0, c1, [&](long long e, auto w) {
    constexpr int W = decltype(w)::value;
    float v[W];
    if constexpr (W == 1) v[0] = QIo<T>::ld1(t.x, e); else QIo<T>::ldv(t.x, e, v);
#pragma unroll
    for (int j = 0; j < W; ++j) {
      float x = isnan(v[j]) ? INFINITY : v[j];
      if (half) x = fmaxf(fminf(x, 65504.f), -65504.f);
      const float a = fabsf(x);
      p.sabs += (double)a;
      p.ssq += (double)x * (double)x;
      p.sat += a >= satv;
      p.ftz += x != 0.f && a < ftzv;
      p.vmax = fmaxf(p.vmax, a);
    }
  });
  return p;
}

__device__ __forceinline__ void q_add(QPart& a, const QPart& b) {
  a.sabs += b.sabs; a.ssq += b.ssq; a.sat += b.sat; a.ftz += b.ftz; a.vmax = fmaxf(a.vmax, b.vmax);
}

__device__ __forceinline__ QPart q_shfl(const QPart& p, int o) {
  QPart q;
  q.sabs = __shfl_xor_sync(0xffffffffu, p.sabs, o);
  q.ssq = __shfl_xor_sync(0xffffffffu, p.ssq, o);
  q.sat = __shfl_xor_sync(0xffffffffu, p.sat, o);
  q.ftz = __shfl_xor_sync(0xffffffffu, p.ftz, o);
  q.vmax = __shfl_xor_sync(0xffffffffu, p.vmax, o);
  return q;
}

// the xor-shuffle tree in every warp, then warp 0 adds the warps' results in order; valid in thread 0
__device__ __forceinline__ QPart q_block_sum(QPart p) {
  __shared__ QPart red[Q_THREADS / 32];
#pragma unroll
  for (int o = 16; o; o >>= 1) q_add(p, q_shfl(p, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = p;
  __syncthreads();
  if (threadIdx.x == 0) {
    p = red[0];
    for (int w = 1; w < Q_THREADS / 32; ++w) q_add(p, red[w]);
  }
  return p;
}

template <typename T>
__global__ void __launch_bounds__(Q_THREADS) q_stats(const __grid_constant__ QTable tab, const QStatConsts k,
                                                     QPart* parts) {
  const QTensor& t = tab.t[q_find(tab, blockIdx.x)];
  const long long c0 = (long long)(blockIdx.x - t.chunk0) * Q_CHUNK;
  const long long c1 = min(c0 + Q_CHUNK, t.size);
  float satv = k.sat_val, ftzv = k.ftz_val;
  if (t.exp) {
    const QFormat f = q_format(*t.exp, k.ebits, k.fbits, k.denorm);
    satv = f.max_float;
    ftzv = f.ftz_float;
  }
  QPart p = t.vec ? q_stats_tensor<T, true>(t, c0, c1, satv, ftzv, k.half)
                  : q_stats_tensor<T, false>(t, c0, c1, satv, ftzv, k.half);
  p = q_block_sum(p);
  if (threadIdx.x == 0) parts[blockIdx.x] = p;
}

// One CTA per tensor: its chunks' parts in chunk order, then the five statistics and, in quantize mode, the exponent
// for the next quantize: from max |x| (mode 0) or mean + stdv * stdv_mul in fp32 (mode 1), plus bias_pad.
__global__ void __launch_bounds__(Q_THREADS) q_stats_finish(const __grid_constant__ QTable tab, const QStatConsts k,
                                                            const QPart* parts) {
  const QTensor& t = tab.t[blockIdx.x];
  const int chunks = (int)((t.size + Q_CHUNK - 1) / Q_CHUNK);
  QPart p = {0.0, 0.0, 0ull, 0ull, 0.f};
  for (int c = threadIdx.x; c < chunks; c += Q_THREADS) q_add(p, parts[t.chunk0 + c]);
  p = q_block_sum(p);
  if (threadIdx.x != 0) return;
  const double n = (double)t.size, mean = p.sabs / n, var = fmax(__dsub_rn(p.ssq / n, __dmul_rn(mean, mean)), 0.0);
  float* s = k.stats + t.index * Q_STATS;
  const float mean_f = (float)mean, stdv_f = (float)sqrt(var);
  s[0] = mean_f;
  s[1] = stdv_f;
  s[2] = (float)(100.0 * (double)p.sat / n);
  s[3] = (float)(100.0 * (double)p.ftz / n);
  s[4] = p.vmax;
  if (t.exp) {
    const float mm = k.mode ? __fadd_rn(mean_f, __fmul_rn(stdv_f, k.stdv_mul)) : p.vmax;
    const int e = ((int)__float_as_uint(mm) >> 23) - 127 + k.bias_pad;
    *t.exp = q_biased(e, k.ebits) - 127;
  }
}

// ---- host side -------------------------------------------------------------------------------------------------------
inline long long q_chunks(long long size) { return (size + Q_CHUNK - 1) / Q_CHUNK; }

// Splits the non-empty tensors into launches of at most Q_MAX tensors and 2^31 - 1 chunks; fill(i, entry) sets the
// pointers of tensor i, launch(table, chunks, first chunk of the call) enqueues the kernels.
template <typename Fill, typename Launch>
inline int q_for_launches(int n, const long long* sizes, Fill&& fill, Launch&& launch) {
  QTable tab;
  tab.n = 0;
  long long chunks = 0, base = 0;
  for (int i = 0; i <= n; ++i) {
    const long long c = i < n ? q_chunks(sizes[i]) : 0;
    if (tab.n && (i == n || tab.n == Q_MAX || chunks + c > 0x7fffffffLL)) {
      if (int e = launch(tab, (int)chunks, base)) return e;
      base += chunks;
      tab.n = 0;
      chunks = 0;
    }
    if (i == n || c == 0) continue;
    QTensor& t = tab.t[tab.n++];
    t = QTensor{};
    t.size = sizes[i];
    t.index = i;
    t.chunk0 = (int)chunks;
    fill(i, t);
    chunks += c;
  }
  return 0;
}

}  // namespace bsmm
