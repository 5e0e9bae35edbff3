// Dense row softmax, its gradient and the top-k family (bst_dense_softmax, bst_dense_softmax_grad, bst_topk_softmax,
// bst_topk in include/bsmm_b200.h).
//
// x is (D0, D1, D2, D3), softmax runs along D3. The optional fp32 mask is (1|D1, 1|D2, D3) with element strides
// (M1, M2, 1); a stride of 0 broadcasts. These ops move bytes and compute almost nothing, so the kernels are built
// around HBM traffic:
//   * rows of <= 1024 entries: one warp per row, <= 8192: one 256-thread CTA per row; either way the row stays in
//     registers between max, exp, sum and store, so x is read once and y written once;
//   * longer rows: one CTA per row, an online max / sum pass, then a write pass that reads x again;
//   * 16-byte loads and stores where every row start is 16-byte aligned (aligned base pointers, D3 a multiple of the
//     vector width), one element per access otherwise;
//   * rows that share a mask row are scheduled back to back (DenseRowMap), so a (1, 1, ctx, ctx) mask comes from HBM
//     about once per call while x and y stream past with evict-first hints.
// Sums are formed in a fixed order (each thread in index order, then the xor-shuffle tree, then the warps in order),
// so results are bitwise reproducible.
#pragma once
#include <float.h>
#include "common.cuh"

namespace bsmm {

constexpr int DSM_WARP_MAX = 1024;      // longest row of the warp-per-row route (32 values per lane)
constexpr int DSM_CTA_THREADS = 256;
constexpr int DSM_CTA_MAX = 8192;       // longest row the CTA route keeps in registers (32 values per thread)
constexpr int DSM_WARPS = 4;            // rows per CTA on the warp route
constexpr int TOPK_MAX = 1024;          // longest row of the top-k family (reference: transformer_op.cc:191)
enum { TOPK_VALUES = 0, TOPK_RECTIFIED = 1, TOPK_REBASE = 2, TOPK_SOFTMAX = 3 };

// Work item w -> (row of x, offset of its mask row). The dims the mask broadcasts over (stride 0; all of them without a
// mask) vary fastest, so the `inner` rows that read one mask row are consecutive work items.
struct DenseRowMap {
  long long D1, D2, M1, M2, inner;
  __device__ __forceinline__ void map(long long w, long long& row, long long& moff) const {
    long long in = w % inner, out = w / inner, d1, d2;
    if (M2 == 0) { d2 = in % D2; in /= D2; } else { d2 = out % D2; out /= D2; }
    if (M1 == 0) { d1 = in % D1; in /= D1; } else { d1 = out; }
    row = (in * D1 + d1) * D2 + d2;
    moff = d1 * M1 + d2 * M2;
  }
};

struct DenseArgs {
  const void* a;          // x (forward, top-k) or dy (gradient)
  const void* b;          // y (gradient)
  const float* mask;      // NULL: no mask
  void* out;              // y (forward, top-k) or dx (gradient)
  int32_t* idx;           // top_k indices (TOPK_VALUES)
  DenseRowMap map;
  long long rows;
  int D3, k, mode;
  float scale;
};

// ---- memory helpers: VEC elements at p (VEC = 1, or a 16-byte chunk); CS = evict-first (data read once) ----------------
template <typename T, int VEC, bool CS>
__device__ __forceinline__ void dsm_ld(const T* p, float (&v)[VEC]) {
  if constexpr (VEC == 1) {
    v[0] = to_f32<T>(CS ? __ldcs(p) : __ldg(p));
  } else {
    static_assert(VEC * sizeof(T) == 16, "16-byte chunks");
    const uint4 u = CS ? __ldcs(reinterpret_cast<const uint4*>(p)) : __ldg(reinterpret_cast<const uint4*>(p));
    const T* e = reinterpret_cast<const T*>(&u);
#pragma unroll
    for (int i = 0; i < VEC; ++i) v[i] = to_f32<T>(e[i]);
  }
}

template <typename T, int VEC>
__device__ __forceinline__ void dsm_st(T* p, const float (&v)[VEC]) {
  if constexpr (VEC == 1) {
    __stcs(p, from_f32<T>(v[0]));
  } else {
    uint4 u;
    T* e = reinterpret_cast<T*>(&u);
#pragma unroll
    for (int i = 0; i < VEC; ++i) e[i] = from_f32<T>(v[i]);
    __stcs(reinterpret_cast<uint4*>(p), u);
  }
}

template <int VEC>
__device__ __forceinline__ void dsm_ld_mask(const float* p, float (&m)[VEC]) {
  if constexpr (VEC == 1) {
    m[0] = __ldg(p);
  } else {
#pragma unroll
    for (int i = 0; i < VEC; i += 4) {
      const float4 f = __ldg(reinterpret_cast<const float4*>(p + i));
      m[i] = f.x; m[i + 1] = f.y; m[i + 2] = f.z; m[i + 3] = f.w;
    }
  }
}

// the softmax argument of one entry (reference transformer.py:609-619): x * m * scale where m != 0, else -FLT_MAX
template <int VEC>
__device__ __forceinline__ void dsm_values(float (&v)[VEC], const float* m, float scale) {
  if (m) {
    float mv[VEC];
    dsm_ld_mask<VEC>(m, mv);
#pragma unroll
    for (int j = 0; j < VEC; ++j) v[j] = mv[j] != 0.f ? v[j] * mv[j] * scale : -FLT_MAX;
  } else {
#pragma unroll
    for (int j = 0; j < VEC; ++j) v[j] *= scale;
  }
}

template <bool MAX> __device__ __forceinline__ float dsm_op(float a, float b) { return MAX ? fmaxf(a, b) : a + b; }

// Max or sum over the `threads` threads of a row (a warp, or the whole CTA); every thread gets the same bits: the xor
// tree adds the same pairs in every lane, the warps' partials are combined in warp order.
template <bool MAX>
__device__ __forceinline__ float dsm_reduce(float v, int threads, float* sh) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v = dsm_op<MAX>(v, __shfl_xor_sync(0xffffffffu, v, o));
  if (threads > 32) {
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
    __syncthreads();
    v = sh[0];
    for (int w = 1; w < threads / 32; ++w) v = dsm_op<MAX>(v, sh[w]);
    __syncthreads();
  }
  return v;
}

// ---- softmax forward ----------------------------------------------------------------------------------------------------
// Register routes: THREADS = 32 (a warp per row, DSM_WARPS rows per CTA) or DSM_CTA_THREADS (a CTA per row). Thread t
// holds the chunks t, t + THREADS, ... (NCH of them, VEC entries each); entries past D3 hold -inf and add exp(-inf) = 0.
template <typename T, int VEC, int NCH, int THREADS>
__global__ void __launch_bounds__(THREADS == 32 ? 32 * DSM_WARPS : THREADS) dense_softmax_kernel(DenseArgs a) {
  __shared__ float sh[32];
  long long w;
  int t;
  if (THREADS == 32) {
    w = (long long)blockIdx.x * DSM_WARPS + (threadIdx.x >> 5);
    t = threadIdx.x & 31;
    if (w >= a.rows) return;                  // whole warps leave; this route has no CTA barrier
  } else {
    w = blockIdx.x;
    t = threadIdx.x;
  }
  long long row, moff;
  a.map.map(w, row, moff);
  const int D3 = a.D3;
  const T* x = reinterpret_cast<const T*>(a.a) + row * D3;
  const float* m = a.mask ? a.mask + moff : nullptr;
  float v[NCH][VEC];
  float mx = -INFINITY;
#pragma unroll
  for (int i = 0; i < NCH; ++i) {
    const int c = (t + i * THREADS) * VEC;
    if (c < D3) {
      dsm_ld<T, VEC, true>(x + c, v[i]);
      dsm_values<VEC>(v[i], m ? m + c : nullptr, a.scale);
    } else {
#pragma unroll
      for (int j = 0; j < VEC; ++j) v[i][j] = -INFINITY;
    }
#pragma unroll
    for (int j = 0; j < VEC; ++j) mx = fmaxf(mx, v[i][j]);
  }
  mx = dsm_reduce<true>(mx, THREADS, sh);
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < NCH; ++i)
#pragma unroll
    for (int j = 0; j < VEC; ++j) { v[i][j] = expf(v[i][j] - mx); s += v[i][j]; }
  s = dsm_reduce<false>(s, THREADS, sh);
  const float inv = 1.f / s;
  T* y = reinterpret_cast<T*>(a.out) + row * D3;
#pragma unroll
  for (int i = 0; i < NCH; ++i) {
    const int c = (t + i * THREADS) * VEC;
    if (c < D3) {
#pragma unroll
      for (int j = 0; j < VEC; ++j) v[i][j] *= inv;
      dsm_st<T, VEC>(y + c, v[i]);
    }
  }
}

// Rows longer than DSM_CTA_MAX: per thread an online (max, sum) over its chunks in index order, the sums rescaled to the
// row max, then a second read of x that writes y. Pass 1 loads with the default policy so that pass 2 can hit L2.
template <typename T, int VEC>
__global__ void __launch_bounds__(DSM_CTA_THREADS) dense_softmax_long_kernel(DenseArgs a) {
  __shared__ float sh[32];
  long long row, moff;
  a.map.map(blockIdx.x, row, moff);
  const int D3 = a.D3;
  const T* x = reinterpret_cast<const T*>(a.a) + row * D3;
  const float* m = a.mask ? a.mask + moff : nullptr;
  float mx = -INFINITY, s = 0.f;
  for (int c = threadIdx.x * VEC; c < D3; c += DSM_CTA_THREADS * VEC) {
    float v[VEC];
    dsm_ld<T, VEC, false>(x + c, v);
    dsm_values<VEC>(v, m ? m + c : nullptr, a.scale);
    float cm = v[0];
#pragma unroll
    for (int j = 1; j < VEC; ++j) cm = fmaxf(cm, v[j]);
    if (cm > mx) { s *= expf(mx - cm); mx = cm; }
#pragma unroll
    for (int j = 0; j < VEC; ++j) s += expf(v[j] - mx);
  }
  const float M = dsm_reduce<true>(mx, DSM_CTA_THREADS, sh);
  s = dsm_reduce<false>(s * expf(mx - M), DSM_CTA_THREADS, sh);
  const float inv = 1.f / s;
  T* y = reinterpret_cast<T*>(a.out) + row * D3;
  for (int c = threadIdx.x * VEC; c < D3; c += DSM_CTA_THREADS * VEC) {
    float v[VEC];
    dsm_ld<T, VEC, true>(x + c, v);
    dsm_values<VEC>(v, m ? m + c : nullptr, a.scale);
#pragma unroll
    for (int j = 0; j < VEC; ++j) v[j] = expf(v[j] - M) * inv;
    dsm_st<T, VEC>(y + c, v);
  }
}

// ---- softmax gradient: dx = (dy - sum_row(dy * y)) * y * m * scale (reference transformer.py:651-656) -----------------
template <int VEC>
__device__ __forceinline__ void dsm_grad_out(float (&d)[VEC], const float (&p)[VEC], float acc, const float* m, float scale) {
  if (m) {
    float mv[VEC];
    dsm_ld_mask<VEC>(m, mv);
#pragma unroll
    for (int j = 0; j < VEC; ++j) d[j] = (d[j] - acc) * p[j] * mv[j] * scale;
  } else {
#pragma unroll
    for (int j = 0; j < VEC; ++j) d[j] = (d[j] - acc) * p[j] * scale;
  }
}

template <typename T, int VEC, int NCH, int THREADS>
__global__ void __launch_bounds__(THREADS == 32 ? 32 * DSM_WARPS : THREADS) dense_softmax_grad_kernel(DenseArgs a) {
  __shared__ float sh[32];
  long long w;
  int t;
  if (THREADS == 32) {
    w = (long long)blockIdx.x * DSM_WARPS + (threadIdx.x >> 5);
    t = threadIdx.x & 31;
    if (w >= a.rows) return;
  } else {
    w = blockIdx.x;
    t = threadIdx.x;
  }
  long long row, moff;
  a.map.map(w, row, moff);
  const int D3 = a.D3;
  const T* dy = reinterpret_cast<const T*>(a.a) + row * D3;
  const T* y = reinterpret_cast<const T*>(a.b) + row * D3;
  float d[NCH][VEC], p[NCH][VEC];
  float acc = 0.f;
#pragma unroll
  for (int i = 0; i < NCH; ++i) {
    const int c = (t + i * THREADS) * VEC;
    if (c < D3) {
      dsm_ld<T, VEC, true>(dy + c, d[i]);
      dsm_ld<T, VEC, true>(y + c, p[i]);
#pragma unroll
      for (int j = 0; j < VEC; ++j) acc += d[i][j] * p[i][j];
    }
  }
  acc = dsm_reduce<false>(acc, THREADS, sh);
  const float* m = a.mask ? a.mask + moff : nullptr;
  T* dx = reinterpret_cast<T*>(a.out) + row * D3;
#pragma unroll
  for (int i = 0; i < NCH; ++i) {
    const int c = (t + i * THREADS) * VEC;
    if (c < D3) {
      dsm_grad_out<VEC>(d[i], p[i], acc, m ? m + c : nullptr, a.scale);
      dsm_st<T, VEC>(dx + c, d[i]);
    }
  }
}

template <typename T, int VEC>
__global__ void __launch_bounds__(DSM_CTA_THREADS) dense_softmax_grad_long_kernel(DenseArgs a) {
  __shared__ float sh[32];
  long long row, moff;
  a.map.map(blockIdx.x, row, moff);
  const int D3 = a.D3;
  const T* dy = reinterpret_cast<const T*>(a.a) + row * D3;
  const T* y = reinterpret_cast<const T*>(a.b) + row * D3;
  float acc = 0.f;
  for (int c = threadIdx.x * VEC; c < D3; c += DSM_CTA_THREADS * VEC) {
    float d[VEC], p[VEC];
    dsm_ld<T, VEC, false>(dy + c, d);
    dsm_ld<T, VEC, false>(y + c, p);
#pragma unroll
    for (int j = 0; j < VEC; ++j) acc += d[j] * p[j];
  }
  acc = dsm_reduce<false>(acc, DSM_CTA_THREADS, sh);
  const float* m = a.mask ? a.mask + moff : nullptr;
  T* dx = reinterpret_cast<T*>(a.out) + row * D3;
  for (int c = threadIdx.x * VEC; c < D3; c += DSM_CTA_THREADS * VEC) {
    float d[VEC], p[VEC];
    dsm_ld<T, VEC, true>(dy + c, d);
    dsm_ld<T, VEC, true>(y + c, p);
    dsm_grad_out<VEC>(d, p, acc, m ? m + c : nullptr, a.scale);
    dsm_st<T, VEC>(dx + c, d);
  }
}

// ---- top-k family: one CTA per row, a bitonic sort of (value, index) keys in shared memory ------------------------------
// key = order-preserving bits of the value (-0 folded into +0) above the complemented index, so a descending sort ranks by
// value descending, then index ascending: a total order. Padding keys are 0, below every real key.
__device__ __forceinline__ unsigned dsm_ord(float f) {
  if (f == 0.f) f = 0.f;
  const unsigned u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float dsm_unord(unsigned o) { return __uint_as_float((o & 0x80000000u) ? (o & 0x7fffffffu) : ~o); }

template <typename T>
__global__ void __launch_bounds__(512) dense_topk_kernel(DenseArgs a, int npow2) {
  __shared__ unsigned long long key[TOPK_MAX];
  __shared__ float outrow[TOPK_MAX];
  __shared__ float sh[32];
  long long row, moff;
  a.map.map(blockIdx.x, row, moff);
  const int D3 = a.D3, k = a.k, tid = threadIdx.x, nt = blockDim.x;
  const T* x = reinterpret_cast<const T*>(a.a) + row * D3;
  const float* m = a.mask ? a.mask + moff : nullptr;
  for (int i = tid; i < npow2; i += nt) {
    unsigned long long kk = 0;
    if (i < D3) {
      float v = to_f32<T>(x[i]);
      if (a.mode == TOPK_SOFTMAX) v = m ? (m[i] != 0.f ? v * m[i] * a.scale : -FLT_MAX) : v * a.scale;
      kk = ((unsigned long long)dsm_ord(v) << 32) | (unsigned)~(unsigned)i;
      outrow[i] = 0.f;
    }
    key[i] = kk;
  }
  __syncthreads();
  for (int size = 2; size <= npow2; size <<= 1) {
    for (int j = size >> 1; j > 0; j >>= 1) {
      for (int i = tid; i < npow2; i += nt) {
        const int p = i ^ j;
        if (p > i) {
          const unsigned long long u = key[i], v = key[p];
          if ((i & size) == 0 ? u < v : u > v) { key[i] = v; key[p] = u; }
        }
      }
      __syncthreads();
    }
  }
  auto index_of = [&](int r) { return (int)~(unsigned)key[r]; };
  if (a.mode == TOPK_VALUES) {
    T* y = reinterpret_cast<T*>(a.out) + row * k;
    int32_t* idx = a.idx + row * k;
    for (int r = tid; r < k; r += nt) {
      const int i = index_of(r);
      y[r] = x[i];                            // a bit-exact copy of the entry
      idx[r] = i;
    }
    return;
  }
  if (a.mode == TOPK_SOFTMAX) {
    const float mx = dsm_unord((unsigned)(key[0] >> 32));
    float s = 0.f;
    for (int r = tid; r < k; r += nt) s += expf(dsm_unord((unsigned)(key[r] >> 32)) - mx);
    s = dsm_reduce<false>(s, nt, sh);
    const float inv = 1.f / s;
    for (int r = tid; r < k; r += nt) outrow[index_of(r)] = expf(dsm_unord((unsigned)(key[r] >> 32)) - mx) * inv;
  } else {
    // reference transformer.py:536-549: top-k entries become max(x, base) - base, base = max(kth value, 0) with rebase
    const float base = a.mode == TOPK_REBASE ? fmaxf(to_f32<T>(x[index_of(k - 1)]), 0.f) : 0.f;
    for (int r = tid; r < k; r += nt) {
      const int i = index_of(r);
      outrow[i] = fmaxf(to_f32<T>(x[i]), base) - base;
    }
  }
  __syncthreads();
  T* y = reinterpret_cast<T*>(a.out) + row * D3;
  for (int i = tid; i < D3; i += nt) y[i] = from_f32<T>(outrow[i]);
}

// ---- softmax cross entropy (bst_softmax_xent, bst_softmax_xent_grad) ------------------------------------------------------
// loss[n] = lse[n] - x[n, label[n]] with lse[n] = logsumexp(x[n, :]); dx[n, j] = dy[n] * (exp(x[n, j] - lse[n]) - [j == label]).
// Nothing is written per element in the forward, so no route keeps a row in registers: every thread runs an online
// (max, sum) over its chunks in index order (xent_unroll chunks loaded before any is used), then the (max, sum) pairs are
// combined across the row. A partial whose entries are all -inf is (m = -inf, s = 0) and must stay so: it never adds
// exp(-inf - (-inf)) = NaN, and it is rescaled to 0 in the combine. A label outside [0, K) makes the row's loss, lse
// and gradient NaN, with no device assert: the label is compared, never used as an address unless it is in range.
struct XentArgs {
  const void* x;          // logits (N, K)
  const void* labels;     // N labels of label_type
  const float* lse_in;    // gradient: the forward's lse
  const float* dy;        // gradient: d(loss)
  float* loss;            // forward
  float* lse;             // forward
  void* dx;               // gradient
  long long rows;
  int K, label_type;
};

__device__ __forceinline__ long long xent_label(const void* p, int type, long long n) {
  switch (type) {
    case BSMM_LABEL_U8:  return __ldg(reinterpret_cast<const uint8_t*>(p) + n);
    case BSMM_LABEL_U16: return __ldg(reinterpret_cast<const uint16_t*>(p) + n);
    case BSMM_LABEL_I32: return __ldg(reinterpret_cast<const int32_t*>(p) + n);
    default:       return __ldg(reinterpret_cast<const long long*>(p) + n);
  }
}

template <int VEC>
constexpr int xent_unroll() { return VEC == 1 ? 8 : 4; }

// Row w and thread t of the row on either route (THREADS = 32: a warp per row, DSM_WARPS rows per CTA).
template <int THREADS>
__device__ __forceinline__ bool xent_row(long long rows, long long& w, int& t) {
  if (THREADS == 32) {
    w = (long long)blockIdx.x * DSM_WARPS + (threadIdx.x >> 5);
    t = threadIdx.x & 31;
    return w < rows;                           // whole warps leave; this route has no CTA barrier
  }
  w = blockIdx.x;
  t = threadIdx.x;
  return true;
}

template <typename T, int VEC, int THREADS>
__global__ void __launch_bounds__(THREADS == 32 ? 32 * DSM_WARPS : THREADS) softmax_xent_kernel(XentArgs a) {
  __shared__ float sh[32];
  constexpr int U = xent_unroll<VEC>();
  constexpr long long STEP = (long long)THREADS * VEC;
  long long n;
  int t;
  if (!xent_row<THREADS>(a.rows, n, t)) return;
  const int K = a.K;
  const T* x = reinterpret_cast<const T*>(a.x) + n * K;
  float mx = -INFINITY, s = 0.f;
  for (long long c0 = (long long)t * VEC; c0 < K; c0 += U * STEP) {
    float v[U][VEC];
#pragma unroll
    for (int u = 0; u < U; ++u)
      if (c0 + u * STEP < K) dsm_ld<T, VEC, true>(x + c0 + u * STEP, v[u]);
#pragma unroll
    for (int u = 0; u < U; ++u) {
      if (c0 + u * STEP >= K) break;
      float cm = v[u][0];
#pragma unroll
      for (int j = 1; j < VEC; ++j) cm = fmaxf(cm, v[u][j]);
      if (cm > mx) { s *= expf(mx - cm); mx = cm; }         // mx = -inf: s is 0 and expf(-inf) = 0
      if (mx != -INFINITY) {
#pragma unroll
        for (int j = 0; j < VEC; ++j) s += expf(v[u][j] - mx);
      } else {
#pragma unroll
        for (int j = 0; j < VEC; ++j) s += v[u][j] != v[u][j] ? v[u][j] : 0.f;   // keep a NaN entry's NaN
      }
    }
  }
  const float M = dsm_reduce<true>(mx, THREADS, sh);
  const float S = dsm_reduce<false>(mx == -INFINITY ? s : s * expf(mx - M), THREADS, sh);
  if (t == 0) {
    const long long lab = xent_label(a.labels, a.label_type, n);
    float lse = M + logf(S), loss = NAN;
    if (lab >= 0 && lab < K) loss = lse - to_f32<T>(x[lab]);
    else lse = NAN;
    a.loss[n] = loss;
    a.lse[n] = lse;
  }
}

template <typename T, int VEC, int THREADS>
__global__ void __launch_bounds__(THREADS == 32 ? 32 * DSM_WARPS : THREADS) softmax_xent_grad_kernel(XentArgs a) {
  constexpr int U = xent_unroll<VEC>();
  constexpr long long STEP = (long long)THREADS * VEC;
  long long n;
  int t;
  if (!xent_row<THREADS>(a.rows, n, t)) return;
  const int K = a.K;
  const long long lab = xent_label(a.labels, a.label_type, n);
  const float dy = __ldg(a.dy + n);
  const float lse = lab >= 0 && lab < K ? __ldg(a.lse_in + n) : NAN;
  const T* x = reinterpret_cast<const T*>(a.x) + n * K;
  T* dx = reinterpret_cast<T*>(a.dx) + n * K;
  for (long long c0 = (long long)t * VEC; c0 < K; c0 += U * STEP) {
    float v[U][VEC];
#pragma unroll
    for (int u = 0; u < U; ++u)
      if (c0 + u * STEP < K) dsm_ld<T, VEC, true>(x + c0 + u * STEP, v[u]);
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const long long c = c0 + u * STEP;
      if (c >= K) break;
#pragma unroll
      for (int j = 0; j < VEC; ++j) v[u][j] = dy * (expf(v[u][j] - lse) - (c + j == lab ? 1.f : 0.f));
      dsm_st<T, VEC>(dx + c, v[u]);
    }
  }
}

// ---- launchers ------------------------------------------------------------------------------------------------------------
template <typename T>
int launch_softmax_xent(const XentArgs& a, bool grad, bool vec, cudaStream_t s) {
  constexpr int V = 16 / sizeof(T);
  const char* name;
  if (a.K <= DSM_WARP_MAX) {
    const unsigned grid = (unsigned)((a.rows + DSM_WARPS - 1) / DSM_WARPS);
    if (grad) {
      if (vec) softmax_xent_grad_kernel<T, V, 32><<<grid, 32 * DSM_WARPS, 0, s>>>(a);
      else     softmax_xent_grad_kernel<T, 1, 32><<<grid, 32 * DSM_WARPS, 0, s>>>(a);
    } else {
      if (vec) softmax_xent_kernel<T, V, 32><<<grid, 32 * DSM_WARPS, 0, s>>>(a);
      else     softmax_xent_kernel<T, 1, 32><<<grid, 32 * DSM_WARPS, 0, s>>>(a);
    }
    name = grad ? "softmax_xent_grad_warp" : "softmax_xent_warp";
  } else {
    const unsigned grid = (unsigned)a.rows;
    if (grad) {
      if (vec) softmax_xent_grad_kernel<T, V, DSM_CTA_THREADS><<<grid, DSM_CTA_THREADS, 0, s>>>(a);
      else     softmax_xent_grad_kernel<T, 1, DSM_CTA_THREADS><<<grid, DSM_CTA_THREADS, 0, s>>>(a);
    } else {
      if (vec) softmax_xent_kernel<T, V, DSM_CTA_THREADS><<<grid, DSM_CTA_THREADS, 0, s>>>(a);
      else     softmax_xent_kernel<T, 1, DSM_CTA_THREADS><<<grid, DSM_CTA_THREADS, 0, s>>>(a);
    }
    name = grad ? "softmax_xent_grad_cta" : "softmax_xent_cta";
  }
  return check_launch(name);
}

// vec: every row start of every operand is 16-byte aligned (checked by the caller).
template <typename T>
int launch_dense_softmax(const DenseArgs& a, bool grad, bool vec, cudaStream_t s) {
  constexpr int V = 16 / sizeof(T);
  const char* name;
  if (a.D3 <= DSM_WARP_MAX) {
    const unsigned grid = (unsigned)((a.rows + DSM_WARPS - 1) / DSM_WARPS);
    constexpr int NV = DSM_WARP_MAX / 32 / V;
    if (grad) {
      if (vec) dense_softmax_grad_kernel<T, V, NV, 32><<<grid, 32 * DSM_WARPS, 0, s>>>(a);
      else     dense_softmax_grad_kernel<T, 1, 32, 32><<<grid, 32 * DSM_WARPS, 0, s>>>(a);
    } else {
      if (vec) dense_softmax_kernel<T, V, NV, 32><<<grid, 32 * DSM_WARPS, 0, s>>>(a);
      else     dense_softmax_kernel<T, 1, 32, 32><<<grid, 32 * DSM_WARPS, 0, s>>>(a);
    }
    name = grad ? "dense_softmax_grad_warp" : "dense_softmax_warp";
  } else if (a.D3 <= DSM_CTA_MAX) {
    constexpr int NV = DSM_CTA_MAX / DSM_CTA_THREADS / V, NS = DSM_CTA_MAX / DSM_CTA_THREADS;
    const unsigned grid = (unsigned)a.rows;
    if (grad) {
      if (vec) dense_softmax_grad_kernel<T, V, NV, DSM_CTA_THREADS><<<grid, DSM_CTA_THREADS, 0, s>>>(a);
      else     dense_softmax_grad_kernel<T, 1, NS, DSM_CTA_THREADS><<<grid, DSM_CTA_THREADS, 0, s>>>(a);
    } else {
      if (vec) dense_softmax_kernel<T, V, NV, DSM_CTA_THREADS><<<grid, DSM_CTA_THREADS, 0, s>>>(a);
      else     dense_softmax_kernel<T, 1, NS, DSM_CTA_THREADS><<<grid, DSM_CTA_THREADS, 0, s>>>(a);
    }
    name = grad ? "dense_softmax_grad_cta" : "dense_softmax_cta";
  } else {
    const unsigned grid = (unsigned)a.rows;
    if (grad) {
      if (vec) dense_softmax_grad_long_kernel<T, V><<<grid, DSM_CTA_THREADS, 0, s>>>(a);
      else     dense_softmax_grad_long_kernel<T, 1><<<grid, DSM_CTA_THREADS, 0, s>>>(a);
    } else {
      if (vec) dense_softmax_long_kernel<T, V><<<grid, DSM_CTA_THREADS, 0, s>>>(a);
      else     dense_softmax_long_kernel<T, 1><<<grid, DSM_CTA_THREADS, 0, s>>>(a);
    }
    name = grad ? "dense_softmax_grad_long" : "dense_softmax_long";
  }
  return check_launch(name);
}

template <typename T>
int launch_dense_topk(const DenseArgs& a, cudaStream_t s) {
  int npow2 = 1;
  while (npow2 < a.D3) npow2 <<= 1;
  const int threads = npow2 / 2 < 32 ? 32 : (npow2 / 2 > 512 ? 512 : npow2 / 2);
  dense_topk_kernel<T><<<(unsigned)a.rows, threads, 0, s>>>(a, npow2);
  return check_launch(a.mode == TOPK_SOFTMAX ? "dense_topk_softmax"
                      : a.mode == TOPK_VALUES ? "dense_topk" : "dense_topk_rectified");
}

}  // namespace bsmm
