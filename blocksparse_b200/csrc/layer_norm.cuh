// Layer norm and its gradient (bsmm_layer_norm, bsmm_layer_norm_grad in include/bsmm_b200.h).
//
// y = relu?(xhat * g + b), xhat = (x - mean) * rstd, rstd = rsqrt(var + epsilon), statistics per row of L features.
// Two layouts:
//   * NC (feature axis last): x is (N, K) with K = S * L; row r = n * S + s is the segment s of minibatch row n, so its L
//     features are contiguous at r * L and its gain / bias start at s * L. Routes by L as the dense softmax
//     (dense_softmax.cuh): a warp per row (L <= 1024) and a CTA per row (<= 8192) keep the row in registers, so the forward
//     reads x once and writes y once and the variance is a second pass over registers; longer rows are read again from
//     L2 for each pass.
//   * CN (feature axis 0): x is (K, N), N contiguous, the layout of BlocksparseMatMul(feature_axis=0). A CTA owns a
//     strip of columns and a range of rows; each thread keeps Welford (mean, M2) of its columns over the rows its warp
//     reads, and the warps are merged (Chan) in warp order in shared memory. When the strips alone cannot fill the GPU,
//     the rows are split across CTAs and a second kernel merges the splits' partials in split order.
// The backward writes dx in the pass that reads dy and x, together with fp32 partials of dg and db that one owner
// (a warp, a CTA, a strip) holds exclusively; ln_reduce_partials adds them in a fixed order. The work partition is a
// function of the shape alone, so every output, dg and db included, is bitwise reproducible, and nothing synchronises
// the host.
#pragma once
#include "dense_softmax.cuh"

namespace bsmm {

constexpr int LN_CTA_THREADS = 256;
constexpr int LN_CN_WARPS = 8;             // rows read in parallel by one CN CTA
constexpr int LN_WARP_UNITS = 2048;        // NC backward: target owners of dg / db partials on the warp route
constexpr int LN_CTA_UNITS = 512;          // ... on the CTA and long routes
constexpr int LN_CN_CTAS = 264;            // CN: split the rows until about this many CTAs run
constexpr int LN_CN_MIN_ROWS = 64;         // CN: fewest rows per split

struct LnArgs {
  const void* x;
  const void* dy;           // backward
  const void* g;            // gain and bias, K entries of gdtype each, read as fp32
  const void* b;
  int gdtype;
  void* y;                  // forward: y; backward: dx
  float* mean;              // one per (segment, row): NC [N][S], CN [N]
  float* rstd;
  float* ws;                // workspace (bsmm_layer_norm_workspace_bytes)
  long long N;              // rows (NC) or columns (CN)
  int K, L, S;              // features, features per segment, segments
  float eps;
  int relu;
  int rpu, units;           // NC backward: rows per partial owner, owners (chunks of rows) per segment
  int splits, rps;          // CN: row splits and rows per split
};

__device__ __forceinline__ float ln_gb(const void* p, int gdtype, long long k) {
  switch (gdtype) {
    case BSMM_F16:  return __half2float(__ldg(reinterpret_cast<const __half*>(p) + k));
    case BSMM_BF16: return __bfloat162float(__ldg(reinterpret_cast<const __nv_bfloat16*>(p) + k));
    default:        return __ldg(reinterpret_cast<const float*>(p) + k);
  }
}

__device__ __forceinline__ float ln_act(float v, int relu) { return relu ? fmaxf(v, 0.f) : v; }

// ---- NC forward -----------------------------------------------------------------------------------------------------------
// THREADS = 32: a warp per row, DSM_WARPS rows per CTA; else a CTA per row. Thread t holds chunks t, t + THREADS, ...
template <typename T, int VEC, int NCH, int THREADS>
__global__ void __launch_bounds__(THREADS == 32 ? 32 * DSM_WARPS : THREADS) ln_nc_fwd_kernel(LnArgs a) {
  __shared__ float sh[32];
  long long r;
  int t;
  if (!xent_row<THREADS>(a.N * a.S, r, t)) return;
  const int L = a.L;
  const T* x = reinterpret_cast<const T*>(a.x) + r * L;
  float v[NCH][VEC];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < NCH; ++i) {
    const int c = (t + i * THREADS) * VEC;
    if (c < L) {
      dsm_ld<T, VEC, true>(x + c, v[i]);
#pragma unroll
      for (int j = 0; j < VEC; ++j) s += v[i][j];
    }
  }
  const float mean = dsm_reduce<false>(s, THREADS, sh) / (float)L;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < NCH; ++i)
    if ((t + i * THREADS) * VEC < L)
#pragma unroll
      for (int j = 0; j < VEC; ++j) { const float d = v[i][j] - mean; q += d * d; }
  const float rstd = rsqrtf(dsm_reduce<false>(q, THREADS, sh) / (float)L + a.eps);
  const int goff = (int)(r % a.S) * L;
  T* y = reinterpret_cast<T*>(a.y) + r * L;
#pragma unroll
  for (int i = 0; i < NCH; ++i) {
    const int c = (t + i * THREADS) * VEC;
    if (c < L) {
#pragma unroll
      for (int j = 0; j < VEC; ++j)
        v[i][j] = ln_act((v[i][j] - mean) * rstd * ln_gb(a.g, a.gdtype, goff + c + j) + ln_gb(a.b, a.gdtype, goff + c + j), a.relu);
      dsm_st<T, VEC>(y + c, v[i]);
    }
  }
  if (t == 0) { a.mean[r] = mean; a.rstd[r] = rstd; }
}

// Rows longer than DSM_CTA_MAX: the sum, the centred sum of squares and the output are three passes over x; the first two
// load with the default policy so that the later passes can hit L2.
template <typename T, int VEC>
__global__ void __launch_bounds__(LN_CTA_THREADS) ln_nc_fwd_long_kernel(LnArgs a) {
  __shared__ float sh[32];
  const long long r = blockIdx.x;
  const int L = a.L;
  const T* x = reinterpret_cast<const T*>(a.x) + r * L;
  float s = 0.f, q = 0.f;
  for (int c = threadIdx.x * VEC; c < L; c += LN_CTA_THREADS * VEC) {
    float v[VEC];
    dsm_ld<T, VEC, false>(x + c, v);
#pragma unroll
    for (int j = 0; j < VEC; ++j) s += v[j];
  }
  const float mean = dsm_reduce<false>(s, LN_CTA_THREADS, sh) / (float)L;
  for (int c = threadIdx.x * VEC; c < L; c += LN_CTA_THREADS * VEC) {
    float v[VEC];
    dsm_ld<T, VEC, false>(x + c, v);
#pragma unroll
    for (int j = 0; j < VEC; ++j) { const float d = v[j] - mean; q += d * d; }
  }
  const float rstd = rsqrtf(dsm_reduce<false>(q, LN_CTA_THREADS, sh) / (float)L + a.eps);
  const int goff = (int)(r % a.S) * L;
  T* y = reinterpret_cast<T*>(a.y) + r * L;
  for (int c = threadIdx.x * VEC; c < L; c += LN_CTA_THREADS * VEC) {
    float v[VEC];
    dsm_ld<T, VEC, true>(x + c, v);
#pragma unroll
    for (int j = 0; j < VEC; ++j)
      v[j] = ln_act((v[j] - mean) * rstd * ln_gb(a.g, a.gdtype, goff + c + j) + ln_gb(a.b, a.gdtype, goff + c + j), a.relu);
    dsm_st<T, VEC>(y + c, v);
  }
  if (threadIdx.x == 0) { a.mean[r] = mean; a.rstd[r] = rstd; }
}

// ---- NC backward ----------------------------------------------------------------------------------------------------------
// dy' = relu ? dy * [xhat g + b > 0] : dy; dyg = dy' g; dx = rstd (dyg - (xhat sum(dyg xhat) + sum(dyg)) / L).
// Owner u = (chunk c, segment s) handles rows n in [c * rpu, (c + 1) * rpu) of segment s and writes its sums of dy' xhat
// and dy' over them to ws[c][s * L + f] (dg) and ws[units + c][s * L + f] (db), with units = a.units chunks.
__device__ __forceinline__ void ln_grad_terms(float x, float dy, float g, float b, float mean, float rstd, int relu,
                                              float& xh, float& dyr) {
  xh = (x - mean) * rstd;
  dyr = relu && !(xh * g + b > 0.f) ? 0.f : dy;
}

// The owner's partials and the current row's xhat live in shared memory (ln_nc_bwd_smem bytes per CTA), in slots that
// only one thread touches: no barrier guards them, and no register array has to hold a row.
template <int NCH, int VEC, int THREADS>
constexpr int ln_nc_bwd_smem() { return 3 * NCH * VEC * 32 * (THREADS == 32 ? DSM_WARPS : THREADS / 32) * (int)sizeof(float); }

template <typename T, int VEC, int NCH, int THREADS>
__global__ void __launch_bounds__(THREADS == 32 ? 32 * DSM_WARPS : THREADS, 1) ln_nc_bwd_kernel(LnArgs a) {
  __shared__ float sh[32];
  extern __shared__ float acc[];
  constexpr int SLOTS = NCH * VEC * THREADS;              // padded row length of one owner
  long long u;
  int t;
  if (!xent_row<THREADS>((long long)a.units * a.S, u, t)) return;
  float* ag = acc + (THREADS == 32 ? (threadIdx.x >> 5) * 3 * SLOTS : 0);
  float* ab = ag + SLOTS;
  float* xs = ab + SLOTS;
  const int L = a.L, S = a.S;
  const int c = (int)(u / S), s = (int)(u % S), goff = s * L;
#pragma unroll 2
  for (int i = 0; i < NCH; ++i)
#pragma unroll
    for (int j = 0; j < VEC; ++j) ag[(t + i * THREADS) * VEC + j] = ab[(t + i * THREADS) * VEC + j] = 0.f;
  const long long n0 = (long long)c * a.rpu, n1 = min(n0 + a.rpu, a.N);
  for (long long n = n0; n < n1; ++n) {
    const long long r = n * S + s;
    const T* x = reinterpret_cast<const T*>(a.x) + r * L;
    const T* dy = reinterpret_cast<const T*>(a.dy) + r * L;
    const float mean = __ldg(a.mean + r), rstd = __ldg(a.rstd + r);
    float s1 = 0.f, s2 = 0.f;                              // dy is read again for dx, from L1 / L2
#pragma unroll 2
    for (int i = 0; i < NCH; ++i) {
      const int f = (t + i * THREADS) * VEC;
      if (f < L) {
        float xv[VEC], dv[VEC];
        dsm_ld<T, VEC, true>(x + f, xv);
        dsm_ld<T, VEC, false>(dy + f, dv);
#pragma unroll
        for (int j = 0; j < VEC; ++j) {
          const float g = ln_gb(a.g, a.gdtype, goff + f + j);
          ln_grad_terms(xv[j], dv[j], g, ln_gb(a.b, a.gdtype, goff + f + j), mean, rstd, a.relu, xv[j], dv[j]);
          xs[f + j] = xv[j];
          ag[f + j] += dv[j] * xv[j];
          ab[f + j] += dv[j];
          s1 += dv[j] * g * xv[j];
          s2 += dv[j] * g;
        }
      }
    }
    s1 = dsm_reduce<false>(s1, THREADS, sh);
    s2 = dsm_reduce<false>(s2, THREADS, sh);
    const float invL = 1.f / (float)L;
    T* dx = reinterpret_cast<T*>(a.y) + r * L;
#pragma unroll 2
    for (int i = 0; i < NCH; ++i) {
      const int f = (t + i * THREADS) * VEC;
      if (f < L) {
        float dv[VEC];
        dsm_ld<T, VEC, true>(dy + f, dv);
#pragma unroll
        for (int j = 0; j < VEC; ++j) {
          const float g = ln_gb(a.g, a.gdtype, goff + f + j), xh = xs[f + j];
          const float dr = a.relu && !(xh * g + ln_gb(a.b, a.gdtype, goff + f + j) > 0.f) ? 0.f : dv[j];
          dv[j] = rstd * (dr * g - (xh * s1 + s2) * invL);
        }
        dsm_st<T, VEC>(dx + f, dv);
      }
    }
  }
  float* pg = a.ws + (long long)c * a.K + goff;
  float* pb = a.ws + ((long long)a.units + c) * a.K + goff;
#pragma unroll 2
  for (int i = 0; i < NCH; ++i) {
    const int f = (t + i * THREADS) * VEC;
    if (f < L)
#pragma unroll
      for (int j = 0; j < VEC; ++j) { pg[f + j] = ag[f + j]; pb[f + j] = ab[f + j]; }
  }
}

// Rows longer than DSM_CTA_MAX: a CTA per owner; per row one pass for the two sums, one that writes dx and adds to the
// owner's partials in place (each partial entry belongs to one thread of one CTA: no race).
template <typename T, int VEC>
__global__ void __launch_bounds__(LN_CTA_THREADS) ln_nc_bwd_long_kernel(LnArgs a) {
  __shared__ float sh[32];
  const int L = a.L, S = a.S;
  const int c = (int)(blockIdx.x / S), s = (int)(blockIdx.x % S), goff = s * L;
  float* pg = a.ws + (long long)c * a.K + goff;
  float* pb = a.ws + ((long long)a.units + c) * a.K + goff;
  const long long n0 = (long long)c * a.rpu, n1 = min(n0 + a.rpu, a.N);
  for (long long n = n0; n < n1; ++n) {
    const long long r = n * S + s;
    const T* x = reinterpret_cast<const T*>(a.x) + r * L;
    const T* dy = reinterpret_cast<const T*>(a.dy) + r * L;
    const float mean = __ldg(a.mean + r), rstd = __ldg(a.rstd + r);
    float s1 = 0.f, s2 = 0.f;
    for (int f = threadIdx.x * VEC; f < L; f += LN_CTA_THREADS * VEC) {
      float xv[VEC], dv[VEC];
      dsm_ld<T, VEC, false>(x + f, xv);
      dsm_ld<T, VEC, false>(dy + f, dv);
#pragma unroll
      for (int j = 0; j < VEC; ++j) {
        const float g = ln_gb(a.g, a.gdtype, goff + f + j);
        float xh, dr;
        ln_grad_terms(xv[j], dv[j], g, ln_gb(a.b, a.gdtype, goff + f + j), mean, rstd, a.relu, xh, dr);
        s1 += dr * g * xh;
        s2 += dr * g;
      }
    }
    s1 = dsm_reduce<false>(s1, LN_CTA_THREADS, sh);
    s2 = dsm_reduce<false>(s2, LN_CTA_THREADS, sh);
    const float invL = 1.f / (float)L;
    T* dx = reinterpret_cast<T*>(a.y) + r * L;
    for (int f = threadIdx.x * VEC; f < L; f += LN_CTA_THREADS * VEC) {
      float xv[VEC], dv[VEC];
      dsm_ld<T, VEC, true>(x + f, xv);
      dsm_ld<T, VEC, true>(dy + f, dv);
#pragma unroll
      for (int j = 0; j < VEC; ++j) {
        const float g = ln_gb(a.g, a.gdtype, goff + f + j);
        float xh, dr;
        ln_grad_terms(xv[j], dv[j], g, ln_gb(a.b, a.gdtype, goff + f + j), mean, rstd, a.relu, xh, dr);
        pg[f + j] = (n == n0 ? 0.f : pg[f + j]) + dr * xh;
        pb[f + j] = (n == n0 ? 0.f : pb[f + j]) + dr;
        dv[j] = rstd * (dr * g - (xh * s1 + s2) * invL);
      }
      dsm_st<T, VEC>(dx + f, dv);
    }
  }
}

// dg[k] = sum_p part[p][k] and db[k] = sum_p part[parts + p][k], p in order; converted to G (the dtype of g and b).
template <typename G>
__global__ void __launch_bounds__(256) ln_reduce_partials_kernel(const float* part, int parts, int K, void* dg, void* db) {
  const int k = blockIdx.x * 256 + threadIdx.x;
  if (k >= K) return;
  float sg = 0.f, sb = 0.f;
  for (int p = 0; p < parts; ++p) {
    sg += part[(long long)p * K + k];
    sb += part[((long long)parts + p) * K + k];
  }
  reinterpret_cast<G*>(dg)[k] = from_f32<G>(sg);
  reinterpret_cast<G*>(db)[k] = from_f32<G>(sb);
}

// ---- CN (feature axis 0) --------------------------------------------------------------------------------------------------
// CTA (strip, split): columns [strip * 32 * VEC, +32 * VEC), rows [split * rps, +rps). Lane l holds the VEC columns at
// l * VEC; warp w reads rows w, w + LN_CN_WARPS, ... of the range. Columns past N are clamped to N - 1 for loads and
// never stored.
template <int VEC>
struct Welford {
  float n, m[VEC], q[VEC];
};

// (nb, mb, qb) merged into (n, m, q) (Chan et al.); nb = 0 leaves it unchanged.
template <int VEC>
__device__ __forceinline__ void chan_merge(Welford<VEC>& w, float nb, const float* mb, const float* qb) {
  if (nb == 0.f) return;
  const float n = w.n + nb, f = nb / n, h = w.n * f;
#pragma unroll
  for (int j = 0; j < VEC; ++j) {
    const float d = mb[j] - w.m[j];
    w.m[j] += d * f;
    w.q[j] += qb[j] + d * d * h;
  }
  w.n = n;
}

template <typename T, int VEC>
__device__ __forceinline__ void cn_load(const T* p, long long col, long long N, float (&v)[VEC]) {
  if constexpr (VEC == 1) {
    v[0] = to_f32<T>(__ldg(p + min(col, N - 1)));
  } else {
    dsm_ld<T, VEC, false>(p + col, v);       // N % VEC == 0 on this route: a chunk is all in or all out
  }
}

// Forward statistics. splits == 1: the CTA also writes y (a second read of its strip) and mean / rstd. Otherwise it
// writes its (mean, M2) to ws[split][N] and ws[splits + split][N], and ln_cn_merge / ln_cn_apply finish.
template <typename T, int VEC>
__global__ void __launch_bounds__(32 * LN_CN_WARPS) ln_cn_fwd_kernel(LnArgs a) {
  __shared__ float shm[LN_CN_WARPS][32 * VEC], shq[LN_CN_WARPS][32 * VEC], shn[LN_CN_WARPS];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long N = a.N, col = ((long long)blockIdx.x * 32 + lane) * VEC;
  const bool live = col < N;
  const long long cc = live ? col : 0;
  const int k0 = blockIdx.y * a.rps, k1 = min(k0 + a.rps, a.K);
  const T* x = reinterpret_cast<const T*>(a.x);
  Welford<VEC> w;
  w.n = 0.f;
#pragma unroll
  for (int j = 0; j < VEC; ++j) w.m[j] = w.q[j] = 0.f;
  constexpr int U = 4;
  for (int k = k0 + warp; k < k1; k += U * LN_CN_WARPS) {
    float v[U][VEC];
#pragma unroll
    for (int u = 0; u < U; ++u)
      if (k + u * LN_CN_WARPS < k1) cn_load<T, VEC>(x + (long long)(k + u * LN_CN_WARPS) * N, VEC == 1 ? col : cc, N, v[u]);
#pragma unroll
    for (int u = 0; u < U; ++u) {
      if (k + u * LN_CN_WARPS >= k1) break;
      w.n += 1.f;
      const float rn = 1.f / w.n;
#pragma unroll
      for (int j = 0; j < VEC; ++j) {
        const float d = v[u][j] - w.m[j];
        w.m[j] += d * rn;
        w.q[j] += d * (v[u][j] - w.m[j]);
      }
    }
  }
#pragma unroll
  for (int j = 0; j < VEC; ++j) { shm[warp][lane * VEC + j] = w.m[j]; shq[warp][lane * VEC + j] = w.q[j]; }
  if (lane == 0) shn[warp] = w.n;
  __syncthreads();
  if (warp == 0) {
    for (int o = 1; o < LN_CN_WARPS; ++o) chan_merge<VEC>(w, shn[o], &shm[o][lane * VEC], &shq[o][lane * VEC]);
#pragma unroll
    for (int j = 0; j < VEC; ++j) { shm[0][lane * VEC + j] = w.m[j]; shq[0][lane * VEC + j] = w.q[j]; }
  }
  __syncthreads();
  if (a.splits > 1) {
    if (warp == 0 && live)
#pragma unroll
      for (int j = 0; j < VEC; ++j)
        if (col + j < N) {
          a.ws[(long long)blockIdx.y * N + col + j] = w.m[j];
          a.ws[((long long)a.splits + blockIdx.y) * N + col + j] = w.q[j];
        }
    return;
  }
  float mean[VEC], rstd[VEC];
#pragma unroll
  for (int j = 0; j < VEC; ++j) {
    mean[j] = shm[0][lane * VEC + j];
    rstd[j] = rsqrtf(shq[0][lane * VEC + j] / (float)a.K + a.eps);
  }
  if (warp == 0 && live)
#pragma unroll
    for (int j = 0; j < VEC; ++j)
      if (col + j < N) { a.mean[col + j] = mean[j]; a.rstd[col + j] = rstd[j]; }
  if (!live) return;
  T* y = reinterpret_cast<T*>(a.y);
  for (int k = k0 + warp; k < k1; k += LN_CN_WARPS) {
    float v[VEC];
    cn_load<T, VEC>(x + (long long)k * N, col, N, v);
    const float g = ln_gb(a.g, a.gdtype, k), b = ln_gb(a.b, a.gdtype, k);
#pragma unroll
    for (int j = 0; j < VEC; ++j) v[j] = ln_act((v[j] - mean[j]) * rstd[j] * g + b, a.relu);
    dsm_st<T, VEC>(y + (long long)k * N + col, v);
  }
}

// Split route: per column, the splits' (mean, M2) merged in split order (every split but the last holds rps rows).
__global__ void __launch_bounds__(256) ln_cn_merge_kernel(LnArgs a) {
  const long long n = (long long)blockIdx.x * 256 + threadIdx.x;
  if (n >= a.N) return;
  Welford<1> w;
  w.n = 0.f; w.m[0] = w.q[0] = 0.f;
  for (int p = 0; p < a.splits; ++p) {
    const float cnt = (float)(min((p + 1) * a.rps, a.K) - p * a.rps);
    const float m = a.ws[(long long)p * a.N + n], q = a.ws[((long long)a.splits + p) * a.N + n];
    chan_merge<1>(w, cnt, &m, &q);
  }
  a.mean[n] = w.m[0];
  a.rstd[n] = rsqrtf(w.q[0] / (float)a.K + a.eps);
}

template <typename T, int VEC>
__global__ void __launch_bounds__(32 * LN_CN_WARPS) ln_cn_apply_kernel(LnArgs a) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long N = a.N, col = ((long long)blockIdx.x * 32 + lane) * VEC;
  if (col >= N) return;
  const int k0 = blockIdx.y * a.rps, k1 = min(k0 + a.rps, a.K);
  float mean[VEC], rstd[VEC];
#pragma unroll
  for (int j = 0; j < VEC; ++j) {
    const long long cj = min(col + j, N - 1);
    mean[j] = __ldg(a.mean + cj); rstd[j] = __ldg(a.rstd + cj);
  }
  const T* x = reinterpret_cast<const T*>(a.x);
  T* y = reinterpret_cast<T*>(a.y);
  for (int k = k0 + warp; k < k1; k += LN_CN_WARPS) {
    float v[VEC];
    cn_load<T, VEC>(x + (long long)k * N, col, N, v);
    const float g = ln_gb(a.g, a.gdtype, k), b = ln_gb(a.b, a.gdtype, k);
#pragma unroll
    for (int j = 0; j < VEC; ++j) v[j] = ln_act((v[j] - mean[j]) * rstd[j] * g + b, a.relu);
    dsm_st<T, VEC>(y + (long long)k * N + col, v);
  }
}

// Backward, pass 1 over dy and x: per column the sums of dyg xhat and dyg over the CTA's rows (warps combined in warp
// order), written to ws[split][N] and ws[splits + split][N]; per row the sums of dy' xhat and dy' over the strip's columns
// (xor-shuffle tree), written to the dg / db partials at ws[2 splits N + strip K + k] and [... + strips K + strip K + k].
template <typename T, int VEC>
__global__ void __launch_bounds__(32 * LN_CN_WARPS) ln_cn_bwd_sums_kernel(LnArgs a) {
  __shared__ float sh1[LN_CN_WARPS][32 * VEC], sh2[LN_CN_WARPS][32 * VEC];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long N = a.N, col = ((long long)blockIdx.x * 32 + lane) * VEC;
  const bool live = col < N;
  const int k0 = blockIdx.y * a.rps, k1 = min(k0 + a.rps, a.K);
  const long long strips = gridDim.x;
  float* pg = a.ws + 2LL * a.splits * N + (long long)blockIdx.x * a.K;
  float* pb = pg + strips * a.K;
  float mean[VEC], rstd[VEC], s1[VEC], s2[VEC];
#pragma unroll
  for (int j = 0; j < VEC; ++j) {
    const long long cj = min(col + j, N - 1);
    mean[j] = __ldg(a.mean + cj); rstd[j] = __ldg(a.rstd + cj);
    s1[j] = s2[j] = 0.f;
  }
  const T* x = reinterpret_cast<const T*>(a.x);
  const T* dy = reinterpret_cast<const T*>(a.dy);
  for (int k = k0 + warp; k < k1; k += LN_CN_WARPS) {
    float xv[VEC], dv[VEC];
    cn_load<T, VEC>(x + (long long)k * N, live ? col : 0, N, xv);
    cn_load<T, VEC>(dy + (long long)k * N, live ? col : 0, N, dv);
    const float g = ln_gb(a.g, a.gdtype, k), b = ln_gb(a.b, a.gdtype, k);
    float rg = 0.f, rb = 0.f;
#pragma unroll
    for (int j = 0; j < VEC; ++j) {
      float xh, dr;
      ln_grad_terms(xv[j], dv[j], g, b, mean[j], rstd[j], a.relu, xh, dr);
      if (!live || col + j >= N) dr = 0.f;
      rg += dr * xh;
      rb += dr;
      s1[j] += dr * g * xh;
      s2[j] += dr * g;
    }
    rg = dsm_reduce<false>(rg, 32, nullptr);
    rb = dsm_reduce<false>(rb, 32, nullptr);
    if (lane == 0) { pg[k] = rg; pb[k] = rb; }
  }
#pragma unroll
  for (int j = 0; j < VEC; ++j) { sh1[warp][lane * VEC + j] = s1[j]; sh2[warp][lane * VEC + j] = s2[j]; }
  __syncthreads();
  if (warp != 0 || !live) return;
  for (int o = 1; o < LN_CN_WARPS; ++o)
#pragma unroll
    for (int j = 0; j < VEC; ++j) { s1[j] += sh1[o][lane * VEC + j]; s2[j] += sh2[o][lane * VEC + j]; }
#pragma unroll
  for (int j = 0; j < VEC; ++j)
    if (col + j < N) {
      a.ws[(long long)blockIdx.y * N + col + j] = s1[j];
      a.ws[((long long)a.splits + blockIdx.y) * N + col + j] = s2[j];
    }
}

// Backward, pass 2: the column sums of every split added in split order, then dx for the CTA's rows.
template <typename T, int VEC>
__global__ void __launch_bounds__(32 * LN_CN_WARPS) ln_cn_bwd_dx_kernel(LnArgs a) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long N = a.N, col = ((long long)blockIdx.x * 32 + lane) * VEC;
  if (col >= N) return;
  const int k0 = blockIdx.y * a.rps, k1 = min(k0 + a.rps, a.K);
  float mean[VEC], rstd[VEC], s1[VEC], s2[VEC];
  const float invK = 1.f / (float)a.K;
#pragma unroll
  for (int j = 0; j < VEC; ++j) {
    const long long cj = min(col + j, N - 1);
    mean[j] = __ldg(a.mean + cj); rstd[j] = __ldg(a.rstd + cj);
    s1[j] = s2[j] = 0.f;
    for (int p = 0; p < a.splits; ++p) {
      s1[j] += a.ws[(long long)p * N + cj];
      s2[j] += a.ws[((long long)a.splits + p) * N + cj];
    }
  }
  const T* x = reinterpret_cast<const T*>(a.x);
  const T* dy = reinterpret_cast<const T*>(a.dy);
  T* dx = reinterpret_cast<T*>(a.y);
  for (int k = k0 + warp; k < k1; k += LN_CN_WARPS) {
    float xv[VEC], dv[VEC];
    cn_load<T, VEC>(x + (long long)k * N, col, N, xv);
    cn_load<T, VEC>(dy + (long long)k * N, col, N, dv);
    const float g = ln_gb(a.g, a.gdtype, k), b = ln_gb(a.b, a.gdtype, k);
#pragma unroll
    for (int j = 0; j < VEC; ++j) {
      float xh, dr;
      ln_grad_terms(xv[j], dv[j], g, b, mean[j], rstd[j], a.relu, xh, dr);
      dv[j] = rstd[j] * (dr * g - (xh * s1[j] + s2[j]) * invK);
    }
    dsm_st<T, VEC>(dx + (long long)k * N + col, dv);
  }
}

// ---- launchers --------------------------------------------------------------------------------------------------------------
// Partition of the NC backward (shape only): owners of dg / db partials and rows per owner.
inline void ln_nc_partition(long long N, int L, int S, int& rpu, int& units) {
  const long long target = L <= DSM_WARP_MAX ? LN_WARP_UNITS : LN_CTA_UNITS;
  long long r = (N * S + target - 1) / target;
  if (r < 1) r = 1;
  rpu = (int)(r > 0x7fffffff ? 0x7fffffff : r);
  units = (int)((N + rpu - 1) / rpu);
}

// Partition of the CN routes (shape only): row splits so that strips * splits reaches about LN_CN_CTAS.
inline void ln_cn_partition(long long N, int K, int vec, int& splits, int& rps) {
  const long long strips = (N + 32LL * vec - 1) / (32LL * vec);
  long long sp = strips >= LN_CN_CTAS ? 1 : (LN_CN_CTAS + strips - 1) / strips;
  const long long maxsp = (K + LN_CN_MIN_ROWS - 1) / LN_CN_MIN_ROWS;
  if (sp > maxsp) sp = maxsp;
  if (sp < 1) sp = 1;
  rps = (int)((K + sp - 1) / sp);
  splits = (K + rps - 1) / rps;
}

// Floats of workspace either direction needs; on axis 0 the most over the access widths (1, 4 and 8 elements).
inline size_t ln_workspace_floats(int axis, long long N, int K, int S) {
  if (axis == 0) {
    long long most = 0;
    for (int vec : {1, 4, 8}) {
      int splits, rps;
      ln_cn_partition(N, K, vec, splits, rps);
      const long long strips = (N + 32LL * vec - 1) / (32LL * vec), f = 2LL * splits * N + 2LL * strips * K;
      if (f > most) most = f;
    }
    return (size_t)most;
  }
  int rpu, units;
  ln_nc_partition(N, K / S, S, rpu, units);
  return (size_t)2 * units * K;
}

template <typename T, int VEC, int NCH, int THREADS>
void ln_nc_bwd_launch(unsigned grid, const LnArgs& a, cudaStream_t s) {
  constexpr int smem = ln_nc_bwd_smem<NCH, VEC, THREADS>();
  // per call: the attribute belongs to the current device
  cudaFuncSetAttribute(ln_nc_bwd_kernel<T, VEC, NCH, THREADS>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  ln_nc_bwd_kernel<T, VEC, NCH, THREADS><<<grid, THREADS == 32 ? 32 * DSM_WARPS : THREADS, smem, s>>>(a);
}

template <typename T>
int launch_layer_norm_nc(LnArgs& a, bool grad, bool vec, int gdtype, void* dg, void* db, cudaStream_t s) {
  constexpr int V = 16 / sizeof(T);
  const long long rows = a.N * a.S;
  const char* name;
  if (grad) ln_nc_partition(a.N, a.L, a.S, a.rpu, a.units);
  const long long work = grad ? (long long)a.units * a.S : rows;
  if (a.L <= DSM_WARP_MAX) {
    constexpr int NV = DSM_WARP_MAX / 32 / V;
    const unsigned grid = (unsigned)((work + DSM_WARPS - 1) / DSM_WARPS);
    if (grad) {
      if (vec) ln_nc_bwd_launch<T, V, NV, 32>(grid, a, s);
      else     ln_nc_bwd_launch<T, 1, 32, 32>(grid, a, s);
    } else {
      if (vec) ln_nc_fwd_kernel<T, V, NV, 32><<<grid, 32 * DSM_WARPS, 0, s>>>(a);
      else     ln_nc_fwd_kernel<T, 1, 32, 32><<<grid, 32 * DSM_WARPS, 0, s>>>(a);
    }
    name = grad ? "layer_norm_grad_nc_warp" : "layer_norm_nc_warp";
  } else if (a.L <= DSM_CTA_MAX) {
    constexpr int NV = DSM_CTA_MAX / LN_CTA_THREADS / V, NS = DSM_CTA_MAX / LN_CTA_THREADS;
    const unsigned grid = (unsigned)work;
    if (grad) {
      if (vec) ln_nc_bwd_launch<T, V, NV, LN_CTA_THREADS>(grid, a, s);
      else     ln_nc_bwd_launch<T, 1, NS, LN_CTA_THREADS>(grid, a, s);
    } else {
      if (vec) ln_nc_fwd_kernel<T, V, NV, LN_CTA_THREADS><<<grid, LN_CTA_THREADS, 0, s>>>(a);
      else     ln_nc_fwd_kernel<T, 1, NS, LN_CTA_THREADS><<<grid, LN_CTA_THREADS, 0, s>>>(a);
    }
    name = grad ? "layer_norm_grad_nc_cta" : "layer_norm_nc_cta";
  } else {
    const unsigned grid = (unsigned)work;
    if (grad) {
      if (vec) ln_nc_bwd_long_kernel<T, V><<<grid, LN_CTA_THREADS, 0, s>>>(a);
      else     ln_nc_bwd_long_kernel<T, 1><<<grid, LN_CTA_THREADS, 0, s>>>(a);
    } else {
      if (vec) ln_nc_fwd_long_kernel<T, V><<<grid, LN_CTA_THREADS, 0, s>>>(a);
      else     ln_nc_fwd_long_kernel<T, 1><<<grid, LN_CTA_THREADS, 0, s>>>(a);
    }
    name = grad ? "layer_norm_grad_nc_long" : "layer_norm_nc_long";
  }
  if (grad) {
    if (int e = check_launch(name)) return e;
    BSMM_DISPATCH_DTYPE(gdtype, G, {
      ln_reduce_partials_kernel<G><<<(unsigned)((a.K + 255) / 256), 256, 0, s>>>(a.ws, a.units, a.K, dg, db);
    });
  }
  return check_launch(name);
}

template <typename T>
int launch_layer_norm_cn(LnArgs& a, bool grad, bool vec, int gdtype, void* dg, void* db, cudaStream_t s) {
  constexpr int V = 16 / sizeof(T);
  const int vw = vec ? V : 1;
  ln_cn_partition(a.N, a.K, vw, a.splits, a.rps);
  const dim3 grid((unsigned)((a.N + 32LL * vw - 1) / (32LL * vw)), (unsigned)a.splits);
  const char* name;
  if (!grad) {
    if (vec) ln_cn_fwd_kernel<T, V><<<grid, 32 * LN_CN_WARPS, 0, s>>>(a);
    else     ln_cn_fwd_kernel<T, 1><<<grid, 32 * LN_CN_WARPS, 0, s>>>(a);
    name = "layer_norm_cn";
    if (a.splits > 1) {
      if (int e = check_launch(name)) return e;
      ln_cn_merge_kernel<<<(unsigned)((a.N + 255) / 256), 256, 0, s>>>(a);
      if (vec) ln_cn_apply_kernel<T, V><<<grid, 32 * LN_CN_WARPS, 0, s>>>(a);
      else     ln_cn_apply_kernel<T, 1><<<grid, 32 * LN_CN_WARPS, 0, s>>>(a);
      name = "layer_norm_cn_split";
    }
    return check_launch(name);
  }
  if (vec) ln_cn_bwd_sums_kernel<T, V><<<grid, 32 * LN_CN_WARPS, 0, s>>>(a);
  else     ln_cn_bwd_sums_kernel<T, 1><<<grid, 32 * LN_CN_WARPS, 0, s>>>(a);
  name = a.splits > 1 ? "layer_norm_grad_cn_split" : "layer_norm_grad_cn";
  if (int e = check_launch(name)) return e;
  if (vec) ln_cn_bwd_dx_kernel<T, V><<<grid, 32 * LN_CN_WARPS, 0, s>>>(a);
  else     ln_cn_bwd_dx_kernel<T, 1><<<grid, 32 * LN_CN_WARPS, 0, s>>>(a);
  BSMM_DISPATCH_DTYPE(gdtype, G, {
    ln_reduce_partials_kernel<G><<<(unsigned)((a.K + 255) / 256), 256, 0, s>>>(a.ws + 2LL * a.splits * a.N, (int)grid.x,
                                                                                  a.K, dg, db);
  });
  return check_launch(name);
}

}  // namespace bsmm
