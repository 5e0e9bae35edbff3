// Elementwise math, casts, filters, sums, concrete gates, gathers and column maxima (bsmm_ew_forward,
// bsmm_ew_backward, bsmm_gain_mul_grad, bsmm_float_cast, bsmm_filter_tensor, bsmm_add_n, bsmm_concrete_gate(_grad,
// _infer), bsmm_fancy_gather(_grad), bsmm_reduce_max(_grad) in include/bsmm_b200.h).
//
// These ops move bytes and compute almost nothing, so each kernel streams its inputs once and its outputs once. Thread t
// of the grid owns the VEC-element chunks t, t + G, ... (G the grid's thread count) with 16-byte accesses when every
// pointer is 16-byte aligned; the n % VEC elements past the last chunk go to the first threads one at a time
// (ew_for). Values are formed in fp32 with the accurate libm functions (expf, logf, tanhf, IEEE division and square
// root; never the approximate intrinsics) and each output is rounded once. No kernel here reduces across threads except
// the gain-mul gradient, whose dg partials follow bias_act_nc_kernel's fixed partition (ewops.cuh) and go through
// bias_grad_reduce_kernel, so dg, like bias_relu's db, is bitwise reproducible.
#pragma once
#include <stdint.h>
#include <type_traits>
#include "ewops.cuh"

namespace bsmm {

// The reference's op codes (blocksparse/ewops.py:25-44).
enum {
  EW_ADD = 0, EW_SUB, EW_MUL, EW_DIV, EW_MAXIMUM, EW_MINIMUM, EW_NEG, EW_RCP, EW_SQR, EW_SQRT, EW_EXP, EW_LOG, EW_SIG,
  EW_TANH, EW_RELU, EW_ELU, EW_GELU, EW_SWISH, EW_BIASADD, EW_GAINMUL, EW_NOPS
};
constexpr float EW_SQRT_2_PI = 0.7978845608028654f;
constexpr int EW_MAX_GRID = 65536 * 4;   // grid-stride beyond this many CTAs
constexpr int ADDN_MAX = 8;

__host__ __device__ constexpr bool ew_binary(int op) { return op <= EW_MINIMUM; }
__host__ __device__ constexpr bool ew_bcast(int op) { return op == EW_BIASADD || op == EW_GAINMUL; }
// the gradients that read z = op(x) instead of x (reference ewops.py:140)
__host__ __device__ constexpr bool ew_grad_reads_z(int op) { return op == EW_SIG || op == EW_TANH || op == EW_RELU; }

struct EwArgs {
  const void* x;    // forward: x; backward: x, or z for ew_grad_reads_z
  const void* y;    // binary ops: y
  const void* b;    // broadcast ops: K entries of bdt
  const void* dz;   // backward
  void* z;          // forward: z; backward: dx
  void* dy;         // backward of a binary op: dy
  long long n, K;
  int bdt;
  float alpha;
};

// Calls f(e, width) for every chunk of VEC elements at e, then for the n % VEC elements after the last chunk.
template <int VEC, typename F>
__device__ __forceinline__ void ew_for(long long n, F&& f) {
  const long long t = (long long)blockIdx.x * EW_THREADS + threadIdx.x, G = (long long)gridDim.x * EW_THREADS;
  const long long chunks = n / VEC;
  for (long long c = t; c < chunks; c += G) f(c * VEC, std::integral_constant<int, VEC>());
  if constexpr (VEC > 1) {
    if (chunks * VEC + t < n) f(chunks * VEC + t, std::integral_constant<int, 1>());
  }
}

inline unsigned ew_grid(long long n, int vec) {
  const long long blocks = (n / vec + EW_THREADS - 1) / EW_THREADS;
  return (unsigned)(blocks < 1 ? 1 : blocks < EW_MAX_GRID ? blocks : EW_MAX_GRID);
}

__device__ __forceinline__ float ew_sig(float x) { return 1.f / (1.f + expf(-x)); }

template <int OP>
__device__ __forceinline__ float ew_fwd(float x, float y, float a) {
  if constexpr (OP == EW_ADD || OP == EW_BIASADD) return x + y;
  if constexpr (OP == EW_SUB) return x - y;
  if constexpr (OP == EW_MUL || OP == EW_GAINMUL) return x * y;
  if constexpr (OP == EW_DIV) return x / y;
  if constexpr (OP == EW_MAXIMUM) return fmaxf(x, y);
  if constexpr (OP == EW_MINIMUM) return fminf(x, y);
  if constexpr (OP == EW_NEG) return -x;
  if constexpr (OP == EW_RCP) return 1.f / x;
  if constexpr (OP == EW_SQR) return x * x;
  if constexpr (OP == EW_SQRT) return sqrtf(x);
  if constexpr (OP == EW_EXP) return expf(x);
  if constexpr (OP == EW_LOG) return logf(x);
  if constexpr (OP == EW_SIG) return ew_sig(x);
  if constexpr (OP == EW_TANH) return tanhf(x);
  if constexpr (OP == EW_RELU) return fmaxf(x, 0.f);
  if constexpr (OP == EW_ELU) return x > 0.f ? x : a * expm1f(x);
  if constexpr (OP == EW_GELU) return 0.5f * x * (1.f + tanhf(EW_SQRT_2_PI * (x + a * x * x * x)));
  if constexpr (OP == EW_SWISH) return x * ew_sig(a * x);
  return 0.f;
}

// dx of a unary op from dz and s (x, or z for ew_grad_reads_z); for the binary ops dx (Y = false) or dy (Y = true)
// from dz, x and y. The gradients follow the reference's (ew_op_gpu.h:952-976), written with accurate math.
template <int OP, bool Y = false>
__device__ __forceinline__ float ew_bwd(float dz, float s, float y, float a) {
  if constexpr (OP == EW_MUL) return Y ? dz * s : dz * y;
  if constexpr (OP == EW_DIV) return Y ? -dz * s / (y * y) : dz / y;
  if constexpr (OP == EW_MAXIMUM) return (Y ? y >= s : s >= y) ? dz : 0.f;
  if constexpr (OP == EW_MINIMUM) return (Y ? y <= s : s <= y) ? dz : 0.f;
  if constexpr (OP == EW_RCP) return -dz / (s * s);
  if constexpr (OP == EW_SQR) return 2.f * dz * s;
  if constexpr (OP == EW_SQRT) return 0.5f * dz / sqrtf(s);
  if constexpr (OP == EW_EXP) return dz * expf(s);
  if constexpr (OP == EW_LOG) return dz / s;
  if constexpr (OP == EW_SIG) return dz * (s - s * s);
  if constexpr (OP == EW_TANH) return dz * (1.f - s * s);
  if constexpr (OP == EW_RELU) return s > 0.f ? dz : 0.f;
  if constexpr (OP == EW_ELU) return s > 0.f ? dz : dz * a * (expm1f(s) + 1.f);
  if constexpr (OP == EW_GELU) {
    const float t = tanhf(EW_SQRT_2_PI * (s + a * s * s * s));
    return 0.5f * dz * (1.f + t) + 0.5f * dz * s * (1.f - t * t) * EW_SQRT_2_PI * (1.f + 3.f * a * s * s);
  }
  if constexpr (OP == EW_SWISH) {
    const float g = ew_sig(a * s);
    return dz * (g + a * s * g * (1.f - g));
  }
  return 0.f;
}

// k = e % K, in 32 bits when both fit
__device__ __forceinline__ long long ew_col(long long e, long long K) {
  if (((unsigned long long)e | (unsigned long long)K) >> 32 == 0) return (unsigned)e % (unsigned)K;
  return e % K;
}

template <typename T, int VEC, int OP>
__global__ void __launch_bounds__(EW_THREADS) ew_fwd_kernel(EwArgs a) {
  const T* X = reinterpret_cast<const T*>(a.x);
  const T* Y = reinterpret_cast<const T*>(a.y);
  T* Z = reinterpret_cast<T*>(a.z);
  ew_for<VEC>(a.n, [&](long long e, auto w) {
    constexpr int W = decltype(w)::value;
    float x[W], y[W];
    dsm_ld<T, W, true>(X + e, x);
    if constexpr (ew_binary(OP)) {
      dsm_ld<T, W, true>(Y + e, y);
    } else if constexpr (ew_bcast(OP)) {
      const long long k = ew_col(e, a.K);   // on the vector route K % VEC == 0: a chunk lies in one row
#pragma unroll
      for (int j = 0; j < W; ++j) y[j] = ew_param(a.b, a.bdt, k + j);
    } else {
#pragma unroll
      for (int j = 0; j < W; ++j) y[j] = 0.f;
    }
#pragma unroll
    for (int j = 0; j < W; ++j) x[j] = ew_fwd<OP>(x[j], y[j], a.alpha);
    dsm_st<T, W>(Z + e, x);
  });
}

template <typename T, int VEC, int OP>
__global__ void __launch_bounds__(EW_THREADS) ew_bwd_kernel(EwArgs a) {
  const T* DZ = reinterpret_cast<const T*>(a.dz);
  const T* S = reinterpret_cast<const T*>(a.x);
  const T* Y = reinterpret_cast<const T*>(a.y);
  T* DX = reinterpret_cast<T*>(a.z);
  T* DY = reinterpret_cast<T*>(a.dy);
  ew_for<VEC>(a.n, [&](long long e, auto w) {
    constexpr int W = decltype(w)::value;
    float dz[W], s[W], y[W], dx[W];
    dsm_ld<T, W, true>(DZ + e, dz);
    dsm_ld<T, W, true>(S + e, s);
    if constexpr (ew_binary(OP)) {
      dsm_ld<T, W, true>(Y + e, y);
#pragma unroll
      for (int j = 0; j < W; ++j) {
        dx[j] = ew_bwd<OP, false>(dz[j], s[j], y[j], a.alpha);
        y[j] = ew_bwd<OP, true>(dz[j], s[j], y[j], a.alpha);
      }
      dsm_st<T, W>(DY + e, y);
    } else {
#pragma unroll
      for (int j = 0; j < W; ++j) dx[j] = ew_bwd<OP>(dz[j], s[j], 0.f, a.alpha);
    }
    dsm_st<T, W>(DX + e, dx);
  });
}

#define EW_FWD_CASE(o) case o: ew_fwd_kernel<T, VEC, o><<<grid, EW_THREADS, 0, s>>>(a); break;
#define EW_BWD_CASE(o) case o: ew_bwd_kernel<T, VEC, o><<<grid, EW_THREADS, 0, s>>>(a); break;

template <typename T, int VEC>
void ew_launch(const EwArgs& a, int op, bool grad, cudaStream_t s) {
  const unsigned grid = ew_grid(a.n, VEC);
  if (!grad) {
    switch (op) {
      EW_FWD_CASE(EW_ADD) EW_FWD_CASE(EW_SUB) EW_FWD_CASE(EW_MUL) EW_FWD_CASE(EW_DIV) EW_FWD_CASE(EW_MAXIMUM)
      EW_FWD_CASE(EW_MINIMUM) EW_FWD_CASE(EW_NEG) EW_FWD_CASE(EW_RCP) EW_FWD_CASE(EW_SQR) EW_FWD_CASE(EW_SQRT)
      EW_FWD_CASE(EW_EXP) EW_FWD_CASE(EW_LOG) EW_FWD_CASE(EW_SIG) EW_FWD_CASE(EW_TANH) EW_FWD_CASE(EW_RELU)
      EW_FWD_CASE(EW_ELU) EW_FWD_CASE(EW_GELU) EW_FWD_CASE(EW_SWISH) EW_FWD_CASE(EW_BIASADD) EW_FWD_CASE(EW_GAINMUL)
      default: break;
    }
  } else {
    switch (op) {
      EW_BWD_CASE(EW_MUL) EW_BWD_CASE(EW_DIV) EW_BWD_CASE(EW_MAXIMUM) EW_BWD_CASE(EW_MINIMUM) EW_BWD_CASE(EW_RCP)
      EW_BWD_CASE(EW_SQR) EW_BWD_CASE(EW_SQRT) EW_BWD_CASE(EW_EXP) EW_BWD_CASE(EW_LOG) EW_BWD_CASE(EW_SIG)
      EW_BWD_CASE(EW_TANH) EW_BWD_CASE(EW_RELU) EW_BWD_CASE(EW_ELU) EW_BWD_CASE(EW_GELU) EW_BWD_CASE(EW_SWISH)
      default: break;
    }
  }
}
#undef EW_FWD_CASE
#undef EW_BWD_CASE

template <typename T>
int launch_ew(const EwArgs& a, int op, bool grad, bool vec, cudaStream_t s) {
  constexpr int V = 16 / sizeof(T);
  if (vec) ew_launch<T, V>(a, op, grad, s);
  else     ew_launch<T, 1>(a, op, grad, s);
  return check_launch(grad ? "ew_backward" : "ew_forward");
}

// ---- gain-mul gradient: dx = dz * g, dg = column sums of dz * x ----------------------------------------------------
// The partition of bias_act_nc_kernel: thread (p, c) owns the VEC columns at c * VEC and the rows of partial p, which it
// walks in order, adding dz * x; one fp32 partial per (p, column), then bias_grad_reduce_kernel.
template <typename T, int VEC>
__global__ void __launch_bounds__(EW_THREADS) gain_mul_grad_kernel(BrArgs a, const void* dz, int tpr) {
  const int KV = a.K / VEC, cv = blockIdx.x * tpr + threadIdx.x % tpr;
  if (cv >= KV) return;
  const int k0 = cv * VEC, rpc = EW_THREADS / tpr;
  float g[VEC];
#pragma unroll
  for (int j = 0; j < VEC; ++j) g[j] = ew_param(a.b, a.bdt, k0 + j);
  for (long long p = (long long)blockIdx.y * rpc + threadIdx.x / tpr; p < a.parts; p += (long long)gridDim.y * rpc) {
    float s[VEC];
#pragma unroll
    for (int j = 0; j < VEC; ++j) s[j] = 0.f;
    const long long r1 = min(a.N, (p + 1) * a.rp);
#pragma unroll 4
    for (long long r = p * a.rp; r < r1; ++r) {
      const long long off = r * a.K + k0;
      float d[VEC], x[VEC];
      dsm_ld<T, VEC, true>(reinterpret_cast<const T*>(dz) + off, d);
      dsm_ld<T, VEC, true>(reinterpret_cast<const T*>(a.x) + off, x);
#pragma unroll
      for (int j = 0; j < VEC; ++j) {
        s[j] += d[j] * x[j];
        d[j] *= g[j];
      }
      dsm_st<T, VEC>(reinterpret_cast<T*>(a.y) + off, d);
    }
#pragma unroll
    for (int j = 0; j < VEC; ++j) a.part[p * a.K + k0 + j] = s[j];
  }
}

// a: x, b = g (bdt), y = dx, part; dz separately. db goes to dg in g's dtype.
template <typename T>
int launch_gain_mul_grad(BrArgs& a, const void* dz, void* dg, bool vec, cudaStream_t s) {
  constexpr int V = 16 / sizeof(T);
  a.rp = br_rows_per_part(a.N, a.K);
  a.parts = br_parts(1, a.N, a.K);
  const int VEC = vec ? V : 1, KV = a.K / VEC;
  int tpr = 1;
  while (tpr < KV && tpr < EW_THREADS) tpr *= 2;
  const long long rpc = EW_THREADS / tpr, gy = (a.parts + rpc - 1) / rpc;
  const dim3 grid((unsigned)((KV + tpr - 1) / tpr), (unsigned)(gy < 65535 ? gy : 65535));
  if (vec) gain_mul_grad_kernel<T, V><<<grid, EW_THREADS, 0, s>>>(a, dz, tpr);
  else     gain_mul_grad_kernel<T, 1><<<grid, EW_THREADS, 0, s>>>(a, dz, tpr);
  if (int e = check_launch("gain_mul_grad")) return e;
  BSMM_DISPATCH_DTYPE(a.bdt, G, {
    bias_grad_reduce_kernel<G><<<(unsigned)((a.K + 7) / 8), 256, 0, s>>>(a.part, a.parts, 1, a.K, a.K, dg);
  });
  return check_launch("gain_mul_grad");
}

// ---- float_cast -------------------------------------------------------------------------------------------------------
// VEC elements at p as fp32, in 16-byte accesses when VEC * sizeof(T) is a multiple of 16
template <typename T, int VEC>
__device__ __forceinline__ void ew_ldv(const T* p, float (&v)[VEC]) {
  constexpr int PER = VEC == 1 ? 1 : 16 / sizeof(T);
#pragma unroll
  for (int c = 0; c < VEC / PER; ++c) {
    float t[PER];
    dsm_ld<T, PER, true>(p + c * PER, t);
#pragma unroll
    for (int i = 0; i < PER; ++i) v[c * PER + i] = t[i];
  }
}

template <typename T, int VEC>
__device__ __forceinline__ void ew_stv(T* p, const float (&v)[VEC]) {
  constexpr int PER = VEC == 1 ? 1 : 16 / sizeof(T);
#pragma unroll
  for (int c = 0; c < VEC / PER; ++c) {
    float t[PER];
#pragma unroll
    for (int i = 0; i < PER; ++i) t[i] = v[c * PER + i];
    dsm_st<T, PER>(p + c * PER, t);
  }
}

constexpr int CAST_VEC = 8;   // 16 bytes of the 16-bit side, 32 of the fp32 side

template <typename TX, typename TY, int VEC>
__global__ void __launch_bounds__(EW_THREADS) float_cast_kernel(const TX* x, TY* y, long long n) {
  ew_for<VEC>(n, [&](long long e, auto w) {
    constexpr int W = decltype(w)::value;
    float v[W];
    ew_ldv<TX, W>(x + e, v);
    ew_stv<TY, W>(y + e, v);
  });
}

template <typename TX, typename TY>
void cast_launch(const void* x, void* y, long long n, bool vec, cudaStream_t s) {
  const TX* X = reinterpret_cast<const TX*>(x);
  TY* Y = reinterpret_cast<TY*>(y);
  if (vec) float_cast_kernel<TX, TY, CAST_VEC><<<ew_grid(n, CAST_VEC), EW_THREADS, 0, s>>>(X, Y, n);
  else     float_cast_kernel<TX, TY, 1><<<ew_grid(n, 1), EW_THREADS, 0, s>>>(X, Y, n);
}

inline int launch_float_cast(int xdt, int ydt, const void* x, void* y, long long n, bool vec, cudaStream_t s) {
  BSMM_DISPATCH_DTYPE(xdt, TX, { BSMM_DISPATCH_DTYPE(ydt, TY, { cast_launch<TX, TY>(x, y, n, vec, s); }); });
  return check_launch("float_cast");
}

// ---- filter_tensor ----------------------------------------------------------------------------------------------------
// y = saturate(scale * zero_nans(zero_infs(x))), the reference's order (ew_op_gpu.cu:820-841); scale is read from
// scale_ptr when it is given, on the device, so a captured graph sees the value at replay.
struct FilterArgs {
  const void* x;
  void* y;
  const float* scale_ptr;
  long long n;
  float scale, saturate;
  int zero_infs, zero_nans;
};

template <typename T, int VEC>
__global__ void __launch_bounds__(EW_THREADS) filter_kernel(FilterArgs a) {
  const float scale = a.scale_ptr ? __ldg(a.scale_ptr) : a.scale, sat = a.saturate;
  ew_for<VEC>(a.n, [&](long long e, auto w) {
    constexpr int W = decltype(w)::value;
    float v[W];
    dsm_ld<T, W, true>(reinterpret_cast<const T*>(a.x) + e, v);
#pragma unroll
    for (int j = 0; j < W; ++j) {
      float t = v[j];
      if (a.zero_infs && isinf(t)) t = 0.f;
      if (a.zero_nans && isnan(t)) t = 0.f;
      t *= scale;
      if (sat != 0.f) t = fmaxf(fminf(t, sat), -sat);   // fminf / fmaxf: a NaN saturates to +sat, as in the reference
      v[j] = t;
    }
    dsm_st<T, W>(reinterpret_cast<T*>(a.y) + e, v);
  });
}

template <typename T>
int launch_filter(const FilterArgs& a, bool vec, cudaStream_t s) {
  constexpr int V = 16 / sizeof(T);
  if (vec) filter_kernel<T, V><<<ew_grid(a.n, V), EW_THREADS, 0, s>>>(a);
  else     filter_kernel<T, 1><<<ew_grid(a.n, 1), EW_THREADS, 0, s>>>(a);
  return check_launch("filter_tensor");
}

// ---- add_n8 -------------------------------------------------------------------------------------------------------------
// y = ((0 + x0) + x1) + ... in fp32, in list order, rounded once
struct AddNArgs {
  const void* x[ADDN_MAX];
  void* y;
  long long n;
  int count;
};

template <typename T, int VEC>
__global__ void __launch_bounds__(EW_THREADS) add_n_kernel(AddNArgs a) {
  ew_for<VEC>(a.n, [&](long long e, auto w) {
    constexpr int W = decltype(w)::value;
    float s[W];
#pragma unroll
    for (int j = 0; j < W; ++j) s[j] = 0.f;
#pragma unroll
    for (int i = 0; i < ADDN_MAX; ++i) {
      if (i < a.count) {
        float v[W];
        dsm_ld<T, W, true>(reinterpret_cast<const T*>(a.x[i]) + e, v);
#pragma unroll
        for (int j = 0; j < W; ++j) s[j] += v[j];
      }
    }
    dsm_st<T, W>(reinterpret_cast<T*>(a.y) + e, s);
  });
}

template <typename T>
int launch_add_n(const AddNArgs& a, bool vec, cudaStream_t s) {
  constexpr int V = 16 / sizeof(T);
  if (vec) add_n_kernel<T, V><<<ew_grid(a.n, V), EW_THREADS, 0, s>>>(a);
  else     add_n_kernel<T, 1><<<ew_grid(a.n, 1), EW_THREADS, 0, s>>>(a);
  return check_launch("add_n");
}

// ---- concrete gate (hard-concrete L0 gate) ----------------------------------------------------------------------------
// Element e draws u = word e % 4 of Philox4x32-10 with key = seed and counter (e / 4, call), as dropout does, and forms
//   f = fp32(u) 2^-32 (1 - 2 eps) + eps,   c = sig((log f - log(1 - f) + loga) / temp),   gate = clamp(c (b - a) + a, 0, 1)
// with f and the stretch c (b - a) + a rounded at every step (no contraction), so a host can replay them exactly. c is
// stored in fp32 for the gradient. The state's call advances by one after the launch, on the device.
struct GateArgs {
  const void* loga;   // forward / infer: loga; gradient: dgate
  void* gate;         // forward / infer: gate; gradient: dloga
  float* concrete;    // forward: written; gradient: read
  const long long* state;
  long long n;
  float rcp_temp, limit_a, limit_b, epsilon;
};

__device__ __forceinline__ float gate_stretch(float c, const GateArgs& a) {
  return __fadd_rn(__fmul_rn(c, __fsub_rn(a.limit_b, a.limit_a)), a.limit_a);
}

template <typename T>
__global__ void __launch_bounds__(EW_THREADS) concrete_gate_kernel(GateArgs a) {
  const unsigned long long seed = (unsigned long long)a.state[0], call = (unsigned long long)a.state[1];
  const uint2 key = make_uint2((unsigned)seed, (unsigned)(seed >> 32));
  const float scale = __fmul_rn(2.3283064365386962891e-10f, __fsub_rn(1.f, __fmul_rn(2.f, a.epsilon)));
  const long long blocks = (a.n + 3) / 4;
  for (long long g = (long long)blockIdx.x * EW_THREADS + threadIdx.x; g < blocks; g += (long long)gridDim.x * EW_THREADS) {
    const uint4 r = philox4x32_10(make_uint4((unsigned)g, (unsigned)(g >> 32), (unsigned)call, (unsigned)(call >> 32)), key);
    const unsigned u[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const long long e = g * 4 + j;
      if (e < a.n) {
        const float f = __fadd_rn(__fmul_rn((float)u[j], scale), a.epsilon);
        const float x = to_f32<T>(reinterpret_cast<const T*>(a.loga)[e]);
        const float c = ew_sig((logf(f) - logf(1.f - f) + x) * a.rcp_temp);
        a.concrete[e] = c;
        reinterpret_cast<T*>(a.gate)[e] = from_f32<T>(fminf(fmaxf(gate_stretch(c, a), 0.f), 1.f));
      }
    }
  }
}

// dloga = [0 <= stretch <= 1] dgate (b - a) c (1 - c) / temp, with the stretch formed from the stored c as above
template <typename T>
__global__ void __launch_bounds__(EW_THREADS) concrete_gate_grad_kernel(GateArgs a) {
  ew_for<1>(a.n, [&](long long e, auto) {
    const float c = __ldg(a.concrete + e), st = gate_stretch(c, a);
    const float dg = to_f32<T>(reinterpret_cast<const T*>(a.loga)[e]);
    const float d = st >= 0.f && st <= 1.f ? dg : 0.f;
    reinterpret_cast<T*>(a.gate)[e] = from_f32<T>(d * (a.limit_b - a.limit_a) * (c - c * c) * a.rcp_temp);
  });
}

template <typename T>
__global__ void __launch_bounds__(EW_THREADS) concrete_gate_infer_kernel(GateArgs a) {
  ew_for<1>(a.n, [&](long long e, auto) {
    const float x = to_f32<T>(reinterpret_cast<const T*>(a.loga)[e]);
    reinterpret_cast<T*>(a.gate)[e] = from_f32<T>(fminf(fmaxf(gate_stretch(ew_sig(x), a), 0.f), 1.f));
  });
}

// mode 0 forward (then advance the state), 1 gradient, 2 inference
template <typename T>
int launch_concrete_gate(const GateArgs& a, int mode, cudaStream_t s) {
  if (mode == 0) {
    concrete_gate_kernel<T><<<ew_grid((a.n + 3) / 4, 1), EW_THREADS, 0, s>>>(a);
    if (int e = check_launch("concrete_gate")) return e;
    dropout_advance_kernel<<<1, 1, 0, s>>>(const_cast<long long*>(a.state));
    return check_launch("concrete_gate");
  }
  if (mode == 1) concrete_gate_grad_kernel<T><<<ew_grid(a.n, 1), EW_THREADS, 0, s>>>(a);
  else           concrete_gate_infer_kernel<T><<<ew_grid(a.n, 1), EW_THREADS, 0, s>>>(a);
  return check_launch(mode == 1 ? "concrete_gate_grad" : "concrete_gate_infer");
}

// ---- fancy_gather -------------------------------------------------------------------------------------------------------
// x (d0, d1, d2), idx (d0) int32: y[i, j] = x[i, max(idx[i], 0), j], or 0 where that index is >= d1 (the reference
// kernel's rule, ew_op_gpu.cu:1434-1504); the gradient scatters dy back to those rows and writes 0 everywhere else.
// Element copies are bit copies of E, the unsigned integer of the element's size.
template <typename E>
__global__ void __launch_bounds__(EW_THREADS) fancy_gather_kernel(const E* x, const int32_t* idx, E* y, long long d0,
                                                                  long long d1, long long d2) {
  ew_for<1>(d0 * d2, [&](long long o, auto) {
    long long r = o;
    const long long j = drop_divmod(r, d2);
    const long long i1 = max(__ldg(idx + r), 0);
    y[o] = i1 < d1 ? __ldg(x + (r * d1 + i1) * d2 + j) : E(0);
  });
}

template <typename E>
__global__ void __launch_bounds__(EW_THREADS) fancy_gather_grad_kernel(const E* dy, const int32_t* idx, E* dx,
                                                                       long long d0, long long d1, long long d2) {
  ew_for<1>(d0 * d1 * d2, [&](long long o, auto) {
    long long r = o;
    const long long j = drop_divmod(r, d2), i1 = drop_divmod(r, d1);
    dx[o] = max(__ldg(idx + r), 0) == i1 ? __ldg(dy + r * d2 + j) : E(0);
  });
}

inline int launch_fancy_gather(int esize, bool grad, const void* src, const int32_t* idx, void* dst, long long d0,
                               long long d1, long long d2, cudaStream_t s) {
  const long long n = grad ? d0 * d1 * d2 : d0 * d2;
  if (esize == 4) {
    if (grad) fancy_gather_grad_kernel<uint32_t><<<ew_grid(n, 1), EW_THREADS, 0, s>>>(
        (const uint32_t*)src, idx, (uint32_t*)dst, d0, d1, d2);
    else      fancy_gather_kernel<uint32_t><<<ew_grid(n, 1), EW_THREADS, 0, s>>>(
        (const uint32_t*)src, idx, (uint32_t*)dst, d0, d1, d2);
  } else {
    if (grad) fancy_gather_grad_kernel<uint16_t><<<ew_grid(n, 1), EW_THREADS, 0, s>>>(
        (const uint16_t*)src, idx, (uint16_t*)dst, d0, d1, d2);
    else      fancy_gather_kernel<uint16_t><<<ew_grid(n, 1), EW_THREADS, 0, s>>>(
        (const uint16_t*)src, idx, (uint16_t*)dst, d0, d1, d2);
  }
  return check_launch(grad ? "fancy_gather_grad" : "fancy_gather");
}

// ---- reduce_max ---------------------------------------------------------------------------------------------------------
// x (d0, d1, d2) -> y, a (d0, d2): the maximum over d1 and its index, by the reference kernel's rule (ew_op_gpu.cu:
// 1545-1575): start from (-FLT_MAX, 0) and take an entry only when it is strictly greater, so the first maximum wins, a
// NaN is never taken, and a column of NaNs or -inf gives (-FLT_MAX, 0). Any partition of the walk gives the same result
// when partial results combine as (larger value, then smaller index), because every part starts at index 0's value.
__device__ __forceinline__ void rmax_take(float& m, long long& i, float v, long long j) {
  if (v > m || (v == m && j < i)) { m = v; i = j; }
}

// d2 > 1: thread per (i0, i2), walking d1 (consecutive threads read consecutive addresses)
template <typename T, typename A>
__global__ void __launch_bounds__(EW_THREADS) reduce_max_col_kernel(const T* x, T* y, A* am, long long d0, long long d1,
                                                                    long long d2) {
  ew_for<1>(d0 * d2, [&](long long o, auto) {
    long long r = o;
    const long long j = drop_divmod(r, d2);
    const T* p = x + r * d1 * d2 + j;
    float m = -FLT_MAX;
    long long i = 0;
    for (long long k = 0; k < d1; ++k) {
      const float v = to_f32<T>(__ldcs(p + k * d2));
      if (v > m) { m = v; i = k; }
    }
    y[o] = from_f32<T>(m);
    am[o] = (A)i;
  });
}

// d2 == 1 (the last axis): a warp per row, lane l walking k = l, l + 32, ..., then the xor-shuffle tree
template <typename T, typename A>
__global__ void __launch_bounds__(EW_THREADS) reduce_max_row_kernel(const T* x, T* y, A* am, long long d0, long long d1) {
  const int lane = threadIdx.x & 31;
  const long long W = (long long)gridDim.x * (EW_THREADS / 32);
  for (long long r = (long long)blockIdx.x * (EW_THREADS / 32) + (threadIdx.x >> 5); r < d0; r += W) {
    const T* p = x + r * d1;
    float m = -FLT_MAX;
    long long i = 0;
    for (long long k = lane; k < d1; k += 32) {
      const float v = to_f32<T>(__ldcs(p + k));
      if (v > m) { m = v; i = k; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float mv = __shfl_xor_sync(0xffffffffu, m, o);
      const long long iv = __shfl_xor_sync(0xffffffffu, i, o);
      rmax_take(m, i, mv, iv);
    }
    if (lane == 0) {
      y[r] = from_f32<T>(m);
      am[r] = (A)i;
    }
  }
}

// dx[i0, k, i2] = k == a[i0, i2] ? dy[i0, i2] : 0, every element written
template <typename T, typename A>
__global__ void __launch_bounds__(EW_THREADS) reduce_max_grad_kernel(const T* dy, const A* am, T* dx, long long d0,
                                                                     long long d1, long long d2) {
  ew_for<1>(d0 * d1 * d2, [&](long long o, auto) {
    long long r = o;
    const long long j = drop_divmod(r, d2), k = drop_divmod(r, d1);
    const long long q = r * d2 + j;
    dx[o] = (long long)__ldg(am + q) == k ? __ldg(dy + q) : from_f32<T>(0.f);
  });
}

template <typename T, typename A>
int launch_reduce_max_t(bool grad, const void* src, void* am, void* dst, void* y, long long d0, long long d1,
                        long long d2, cudaStream_t s) {
  if (grad) {
    reduce_max_grad_kernel<T, A><<<ew_grid(d0 * d1 * d2, 1), EW_THREADS, 0, s>>>(
        (const T*)src, (const A*)am, (T*)dst, d0, d1, d2);
    return check_launch("reduce_max_grad");
  }
  if (d2 == 1) {
    const long long blocks = (d0 + EW_THREADS / 32 - 1) / (EW_THREADS / 32);
    reduce_max_row_kernel<T, A><<<(unsigned)(blocks < EW_MAX_GRID ? blocks : EW_MAX_GRID), EW_THREADS, 0, s>>>(
        (const T*)src, (T*)y, (A*)am, d0, d1);
    return check_launch("reduce_max_row");
  }
  reduce_max_col_kernel<T, A><<<ew_grid(d0 * d2, 1), EW_THREADS, 0, s>>>((const T*)src, (T*)y, (A*)am, d0, d1, d2);
  return check_launch("reduce_max_col");
}

// forward: src = x, y and am written; gradient: src = dy, am read, dst = dx
template <typename T>
int launch_reduce_max(int idx_type, bool grad, const void* src, void* am, void* dst, void* y, long long d0, long long d1,
                      long long d2, cudaStream_t s) {
  if (idx_type == BSMM_LABEL_U8) return launch_reduce_max_t<T, uint8_t>(grad, src, am, dst, y, d0, d1, d2, s);
  if (idx_type == BSMM_LABEL_U16) return launch_reduce_max_t<T, uint16_t>(grad, src, am, dst, y, d0, d1, d2, s);
  return launch_reduce_max_t<T, int32_t>(grad, src, am, dst, y, d0, d1, d2, s);
}

}  // namespace bsmm
