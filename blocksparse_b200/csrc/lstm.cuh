// LSTM gate nonlinearity, with or without a layer norm fused in front, and sparse relu (bsmm_lstm_gates(_grad),
// bsmm_lstm_ln_gates(_grad), bsmm_sparse_relu, bsmm_relu_mask_grad in include/bsmm_b200.h).
//
// lstm_gates: per element of the (N, K) cell state, with the gates i, u, f, o read at row r from g[j] + r * gs:
//   c_next = sig(f + b_f + forget_bias) c + sig(i + b_i) tanh(u + b_u),  h_next = sig(o + b_o) tanh(c_next).
// The fused (N, 4K) gate tensor is g[j] = h + j K with gs = 4K; four separate tensors have gs = K. Everything is formed
// in fp32 with expf / tanhf (no fast-math intrinsics) and each output is rounded once. The backward recomputes the gates
// from the inputs (nothing is saved) and writes dc and the four gate gradients with the same pointer scheme. Thread
// (p, c) owns the VEC columns at c * VEC and walks rows p, p + P, ... as bias_act_nc_kernel does, so a row count past
// the grid's y limit needs no second launch. Without a bias nothing is added, so the fused and four-tensor forms give
// the same bits.
//
// sparse_relu: y = max(x - (mean + alpha std), 0) per row of K, std the population standard deviation. The statistics
// are two passes in fp32 (the sum, then the centred sum of squares; never E[x^2] - E[x]^2), reduced in a fixed order
// with dsm_reduce, routed by K as the layer norm forward: a warp per row (K <= 1024) and a CTA per row (<= 8192) keep
// the row in registers; longer rows are read three times, the later passes from L2. A row whose entries are all equal
// gives zeros, as its std is exactly 0 (an fp32 mean need not equal the entries it averages). The gradient is relu's on
// the output, an elementwise mask.
#pragma once
#include "ewops.cuh"
#include "layer_norm.cuh"

namespace bsmm {

struct LstmArgs {
  const void* c;        // c_prev, (N, K) contiguous
  const void* g[4];     // i, u, f, o: row r at g[j] + r * gs
  const void* bias;     // NULL, or 4K entries of bdt: the i, u, f, o blocks
  const void* ec;       // backward: incoming gradients of c_next and h_next, (N, K); NULL reads as 0
  const void* eh;
  void* c_out;          // forward: c_next; backward: dc
  void* h_out;          // forward: h_next
  void* dg[4];          // backward: di, du, df, do, laid out as g
  long long N, gs;
  int K, bdt;
  float forget_bias;
};

__device__ __forceinline__ float lstm_sig(float z) { return 1.f / (1.f + expf(-z)); }

// BIAS is a template parameter, not a test of a.bias in the loop: the compiler hoists the loop-invariant __ldg of the
// bias above such a test, which would read through a null pointer.
template <typename T, int VEC, bool GRAD, bool BIAS>
__global__ void __launch_bounds__(EW_THREADS) lstm_gates_kernel(LstmArgs a, int tpr) {
  const int KV = a.K / VEC, cv = blockIdx.x * tpr + threadIdx.x % tpr;
  if (cv >= KV) return;
  const int k0 = cv * VEC, rpc = EW_THREADS / tpr;
  for (long long r = (long long)blockIdx.y * rpc + threadIdx.x / tpr; r < a.N; r += (long long)gridDim.y * rpc) {
    const long long z = r * a.K + k0, x = r * a.gs + k0;
    float c[VEC], v[4][VEC];
    dsm_ld<T, VEC, true>(reinterpret_cast<const T*>(a.c) + z, c);
#pragma unroll
    for (int g = 0; g < 4; ++g) dsm_ld<T, VEC, true>(reinterpret_cast<const T*>(a.g[g]) + x, v[g]);
    float eh[VEC], ec[VEC];
    if constexpr (GRAD) {
#pragma unroll
      for (int j = 0; j < VEC; ++j) eh[j] = ec[j] = 0.f;
      if (a.eh) dsm_ld<T, VEC, true>(reinterpret_cast<const T*>(a.eh) + z, eh);
      if (a.ec) dsm_ld<T, VEC, true>(reinterpret_cast<const T*>(a.ec) + z, ec);
    }
    if constexpr (BIAS) {
#pragma unroll
      for (int g = 0; g < 4; ++g)
#pragma unroll
        for (int j = 0; j < VEC; ++j) v[g][j] += ew_param(a.bias, a.bdt, (long long)g * a.K + k0 + j);
    }
#pragma unroll
    for (int j = 0; j < VEC; ++j) {
      const float si = lstm_sig(v[0][j]), tu = tanhf(v[1][j]);
      const float sf = lstm_sig(v[2][j] + a.forget_bias), so = lstm_sig(v[3][j]);
      const float cn = sf * c[j] + si * tu, tc = tanhf(cn);
      if constexpr (!GRAD) {
        c[j] = cn;
        v[0][j] = so * tc;
      } else {
        // the reference's LSTM_Backward: sig' = s - s s, tanh' = 1 - t t, written in terms of the outputs
        const float dC = eh[j] * so * (1.f - tc * tc) + ec[j];
        v[0][j] = dC * tu * (si - si * si);
        v[1][j] = dC * si * (1.f - tu * tu);
        v[2][j] = dC * c[j] * (sf - sf * sf);
        v[3][j] = eh[j] * tc * (so - so * so);
        c[j] = dC * sf;
      }
    }
    dsm_st<T, VEC>(reinterpret_cast<T*>(a.c_out) + z, c);
    if constexpr (!GRAD) {
      dsm_st<T, VEC>(reinterpret_cast<T*>(a.h_out) + z, v[0]);
    } else {
#pragma unroll
      for (int g = 0; g < 4; ++g) dsm_st<T, VEC>(reinterpret_cast<T*>(a.dg[g]) + x, v[g]);
    }
  }
}

template <typename T, int VEC, bool GRAD>
void lstm_launch(const LstmArgs& a, cudaStream_t s) {
  const int KV = a.K / VEC;
  int tpr = 1;
  while (tpr < KV && tpr < EW_THREADS) tpr *= 2;
  const long long rpc = EW_THREADS / tpr, gy = (a.N + rpc - 1) / rpc;
  const dim3 grid((unsigned)((KV + tpr - 1) / tpr), (unsigned)(gy < 65535 ? gy : 65535));
  if (a.bias) lstm_gates_kernel<T, VEC, GRAD, true><<<grid, EW_THREADS, 0, s>>>(a, tpr);
  else        lstm_gates_kernel<T, VEC, GRAD, false><<<grid, EW_THREADS, 0, s>>>(a, tpr);
}

template <typename T>
int launch_lstm_gates(const LstmArgs& a, bool grad, bool vec, cudaStream_t s) {
  constexpr int V = 16 / sizeof(T);
  if (grad) {
    if (vec) lstm_launch<T, V, true>(a, s);
    else     lstm_launch<T, 1, true>(a, s);
  } else {
    if (vec) lstm_launch<T, V, false>(a, s);
    else     lstm_launch<T, 1, false>(a, s);
  }
  return check_launch(grad ? "lstm_gates_grad" : "lstm_gates");
}

// ---- layer norm fused into the gates ----------------------------------------------------------------------------------
// lstm_ln_gates: row n of z (4K real columns at z + n * zs) is four segments i, u, f, o of K features; each is
// normalised with its own fp32 mean and rstd (two passes: the sum, then the centred sum of squares, as layer_norm's NC
// route), v = xhat g + b is kept in fp32 and goes straight into the gate formulas of lstm_gates_kernel. A CTA owns a
// row at a time; thread t holds columns t, t + LNG_THREADS, ... of every segment, so z is read three times from L1 / L2
// and c once. Scalar accesses: any alignment and any row stride.
//
// The backward writes dc and dz (z's layout) and the fp32 partials of dg and db. CTA p owns rows [p rpu, (p+1) rpu)
// and its partial slots ws[p][4K] (dg) and ws[P + p][4K] (db), the layout ln_reduce_partials_kernel adds in p order. The
// rows are taken LNG_RB at a time: pass A recomputes the gates and their gradient dv per row and reduces the layer
// norm's two row sums (dv g xhat and dv g per segment) into shared memory, writing dc; pass B walks the columns, row by
// row inside each column, writes dz = rstd (dv g - (xhat s1 + s2) / K) and adds dv xhat and dv into the slot in
// registers, touching the slot once per batch. With `accumulate` the first batch adds to what the slot holds, so T
// calls on one stream sum T steps into one buffer; each slot belongs to one thread of one CTA per call: no atomics.
constexpr int LNG_THREADS = 256;
constexpr int LNG_RB = 8;               // rows per batch of the backward
constexpr int LNG_UNITS = 264;          // target owners of dg / db partials (a shape-only constant)
constexpr int LNG_MAX_CTAS = 1 << 20;   // forward rows beyond this many CTAs are walked by a grid-stride loop

struct LnGatesArgs {
  const void* c;        // (N, K) contiguous
  const void* z;        // (N, 4K) at row stride zs
  const void* g;        // 4K entries of gdt each
  const void* b;
  const void* ec;       // backward: NULL reads as 0
  const void* eh;
  void* c_out;          // forward: c_next; backward: dc
  void* h_out;          // forward: h_next; backward: dz (row stride zs)
  float* mean;          // [N][4]
  float* rstd;
  float* ws;            // backward: [2][P][4K]
  long long N, zs;
  int K, gdt, rpu, accumulate;
  float eps, forget_bias;
};

inline void lng_partition(long long N, int& rpu, int& parts) {
  long long r = (N + LNG_UNITS - 1) / LNG_UNITS;
  if (r < 1) r = 1;
  rpu = (int)r;                         // N / 264 < 2^31 for any N < 2^63 / 4
  parts = (int)((N + r - 1) / r);
}

// The four sums of v over the CTA, each in a fixed order (xor tree, then the warps in order); every thread gets the
// same bits.
__device__ __forceinline__ void lng_reduce4(float (&v)[4], float* sh) {
  constexpr int W = LNG_THREADS / 32;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
#pragma unroll
    for (int o = 16; o; o >>= 1) v[j] += __shfl_xor_sync(0xffffffffu, v[j], o);
    if ((threadIdx.x & 31) == 0) sh[j * W + (threadIdx.x >> 5)] = v[j];
  }
  __syncthreads();
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    v[j] = sh[j * W];
    for (int w = 1; w < W; ++w) v[j] += sh[j * W + w];
  }
  __syncthreads();
}

// The normalised gate inputs v and xhat of column k of a row.
template <typename T>
__device__ __forceinline__ void lng_norm(const LnGatesArgs& a, const T* z, int k, const float* mean, const float* rstd,
                                         float (&v)[4], float (&xh)[4], float (&g)[4]) {
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int f = j * a.K + k;
    g[j] = ln_gb(a.g, a.gdt, f);
    xh[j] = (to_f32<T>(__ldg(z + f)) - mean[j]) * rstd[j];
    v[j] = xh[j] * g[j] + ln_gb(a.b, a.gdt, f);
  }
}

template <typename T>
__global__ void __launch_bounds__(LNG_THREADS) lstm_ln_gates_kernel(LnGatesArgs a) {
  __shared__ float sh[4 * LNG_THREADS / 32];
  const int K = a.K;
  for (long long n = blockIdx.x; n < a.N; n += gridDim.x) {
    const T* z = reinterpret_cast<const T*>(a.z) + n * a.zs;
    float mean[4] = {0.f, 0.f, 0.f, 0.f}, rstd[4] = {0.f, 0.f, 0.f, 0.f};
    for (int k = threadIdx.x; k < K; k += LNG_THREADS)
#pragma unroll
      for (int j = 0; j < 4; ++j) mean[j] += to_f32<T>(__ldg(z + j * K + k));
    lng_reduce4(mean, sh);
#pragma unroll
    for (int j = 0; j < 4; ++j) mean[j] /= (float)K;
    for (int k = threadIdx.x; k < K; k += LNG_THREADS)
#pragma unroll
      for (int j = 0; j < 4; ++j) { const float d = to_f32<T>(__ldg(z + j * K + k)) - mean[j]; rstd[j] += d * d; }
    lng_reduce4(rstd, sh);
#pragma unroll
    for (int j = 0; j < 4; ++j) rstd[j] = rsqrtf(rstd[j] / (float)K + a.eps);
    const long long row = n * K;
    for (int k = threadIdx.x; k < K; k += LNG_THREADS) {
      float v[4], xh[4], g[4];
      lng_norm<T>(a, z, k, mean, rstd, v, xh, g);
      const float si = lstm_sig(v[0]), tu = tanhf(v[1]), sf = lstm_sig(v[2] + a.forget_bias), so = lstm_sig(v[3]);
      const float cn = sf * to_f32<T>(__ldg(reinterpret_cast<const T*>(a.c) + row + k)) + si * tu;
      reinterpret_cast<T*>(a.c_out)[row + k] = from_f32<T>(cn);
      reinterpret_cast<T*>(a.h_out)[row + k] = from_f32<T>(so * tanhf(cn));
    }
    if (threadIdx.x == 0)
#pragma unroll
      for (int j = 0; j < 4; ++j) { a.mean[n * 4 + j] = mean[j]; a.rstd[n * 4 + j] = rstd[j]; }
  }
}

// Gradients dv of the gate inputs at column k of row n (the formulas of lstm_gates_kernel's backward); dcp gets dc.
template <typename T>
__device__ __forceinline__ void lng_dv(const LnGatesArgs& a, long long n, int k, const float (&v)[4], float (&dv)[4],
                                       float& dcp) {
  const long long e = n * a.K + k;
  const float c = to_f32<T>(__ldg(reinterpret_cast<const T*>(a.c) + e));
  const float eh = a.eh ? to_f32<T>(__ldg(reinterpret_cast<const T*>(a.eh) + e)) : 0.f;
  const float ec = a.ec ? to_f32<T>(__ldg(reinterpret_cast<const T*>(a.ec) + e)) : 0.f;
  const float si = lstm_sig(v[0]), tu = tanhf(v[1]), sf = lstm_sig(v[2] + a.forget_bias), so = lstm_sig(v[3]);
  const float tc = tanhf(sf * c + si * tu);
  const float dC = eh * so * (1.f - tc * tc) + ec;
  dv[0] = dC * tu * (si - si * si);
  dv[1] = dC * si * (1.f - tu * tu);
  dv[2] = dC * c * (sf - sf * sf);
  dv[3] = eh * tc * (so - so * so);
  dcp = dC * sf;
}

template <typename T>
__global__ void __launch_bounds__(LNG_THREADS) lstm_ln_gates_grad_kernel(LnGatesArgs a) {
  __shared__ float sh[4 * LNG_THREADS / 32];
  __shared__ float rs[LNG_RB][8];       // per row of the batch: s1 and s2 of the four segments
  const int K = a.K, K4 = 4 * K;
  const long long parts = gridDim.x, r0 = (long long)blockIdx.x * a.rpu, r1 = min(r0 + a.rpu, a.N);
  float* pg = a.ws + (long long)blockIdx.x * K4;
  float* pb = a.ws + (parts + blockIdx.x) * K4;
  const float invK = 1.f / (float)K;
  for (long long n0 = r0; n0 < r1; n0 += LNG_RB) {
    const int nb = (int)min((long long)LNG_RB, r1 - n0);
    for (int i = 0; i < nb; ++i) {
      const long long n = n0 + i;
      const T* z = reinterpret_cast<const T*>(a.z) + n * a.zs;
      float mean[4], rstd[4], s1[4] = {0.f, 0.f, 0.f, 0.f}, s2[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
      for (int j = 0; j < 4; ++j) { mean[j] = __ldg(a.mean + n * 4 + j); rstd[j] = __ldg(a.rstd + n * 4 + j); }
      for (int k = threadIdx.x; k < K; k += LNG_THREADS) {
        float v[4], xh[4], g[4], dv[4], dc;
        lng_norm<T>(a, z, k, mean, rstd, v, xh, g);
        lng_dv<T>(a, n, k, v, dv, dc);
        reinterpret_cast<T*>(a.c_out)[n * K + k] = from_f32<T>(dc);
#pragma unroll
        for (int j = 0; j < 4; ++j) { s1[j] += dv[j] * g[j] * xh[j]; s2[j] += dv[j] * g[j]; }
      }
      lng_reduce4(s1, sh);
      lng_reduce4(s2, sh);
      if (threadIdx.x == 0)
#pragma unroll
        for (int j = 0; j < 4; ++j) { rs[i][j] = s1[j]; rs[i][4 + j] = s2[j]; }
    }
    __syncthreads();
    const bool fresh = n0 == r0 && !a.accumulate;
    for (int k = threadIdx.x; k < K; k += LNG_THREADS) {
      float ag[4], ab[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        ag[j] = fresh ? 0.f : pg[j * K + k];
        ab[j] = fresh ? 0.f : pb[j * K + k];
      }
      for (int i = 0; i < nb; ++i) {
        const long long n = n0 + i;
        const T* z = reinterpret_cast<const T*>(a.z) + n * a.zs;
        float mean[4], rstd[4], v[4], xh[4], g[4], dv[4], dc;
#pragma unroll
        for (int j = 0; j < 4; ++j) { mean[j] = __ldg(a.mean + n * 4 + j); rstd[j] = __ldg(a.rstd + n * 4 + j); }
        lng_norm<T>(a, z, k, mean, rstd, v, xh, g);
        lng_dv<T>(a, n, k, v, dv, dc);
        T* dz = reinterpret_cast<T*>(a.h_out) + n * a.zs;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          ag[j] += dv[j] * xh[j];
          ab[j] += dv[j];
          dz[j * K + k] = from_f32<T>(rstd[j] * (dv[j] * g[j] - (xh[j] * rs[i][j] + rs[i][4 + j]) * invK));
        }
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) { pg[j * K + k] = ag[j]; pb[j * K + k] = ab[j]; }
    }
    __syncthreads();                    // rs is rewritten by the next batch
  }
}

template <typename T>
int launch_lstm_ln_gates(LnGatesArgs& a, bool grad, cudaStream_t s) {
  if (!grad) {
    const unsigned grid = (unsigned)(a.N < LNG_MAX_CTAS ? a.N : LNG_MAX_CTAS);
    lstm_ln_gates_kernel<T><<<grid, LNG_THREADS, 0, s>>>(a);
    return check_launch("lstm_ln_gates");
  }
  int parts;
  lng_partition(a.N, a.rpu, parts);
  lstm_ln_gates_grad_kernel<T><<<(unsigned)parts, LNG_THREADS, 0, s>>>(a);
  return check_launch("lstm_ln_gates_grad");
}

// ---- sparse relu ----------------------------------------------------------------------------------------------------
struct SreluArgs {
  const void* x;
  void* y;
  long long N;
  int K;
  float alpha;
};

constexpr int SRELU_MAX_CTAS = 1 << 20;   // rows beyond grid * rows-per-CTA are walked by a grid-stride loop

// Register routes: THREADS = 32 (a warp per row, DSM_WARPS rows per CTA) or DSM_CTA_THREADS (a CTA per row); thread t
// holds the chunks t, t + THREADS, ... (NCH of VEC entries).
template <typename T, int VEC, int NCH, int THREADS>
__global__ void __launch_bounds__(THREADS == 32 ? 32 * DSM_WARPS : THREADS) sparse_relu_kernel(SreluArgs a) {
  __shared__ float sh[32];
  constexpr int PER = THREADS == 32 ? DSM_WARPS : 1;
  const int t = THREADS == 32 ? threadIdx.x & 31 : threadIdx.x, K = a.K;
  for (long long r = (long long)blockIdx.x * PER + (THREADS == 32 ? threadIdx.x >> 5 : 0); r < a.N;
       r += (long long)gridDim.x * PER) {
    const T* x = reinterpret_cast<const T*>(a.x) + r * K;
    const float x0 = to_f32<T>(__ldg(x));
    float v[NCH][VEC];
    float s = 0.f;
    bool differs = false;
#pragma unroll
    for (int i = 0; i < NCH; ++i) {
      const int c = (t + i * THREADS) * VEC;
      if (c < K) {
        dsm_ld<T, VEC, true>(x + c, v[i]);
#pragma unroll
        for (int j = 0; j < VEC; ++j) { s += v[i][j]; differs |= v[i][j] != x0; }
      }
    }
    const float mean = dsm_reduce<false>(s, THREADS, sh) / (float)K;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < NCH; ++i)
      if ((t + i * THREADS) * VEC < K)
#pragma unroll
        for (int j = 0; j < VEC; ++j) { const float d = v[i][j] - mean; q += d * d; }
    const float sd = sqrtf(dsm_reduce<false>(q, THREADS, sh) / (float)K);
    const bool flat = THREADS == 32 ? !__any_sync(0xffffffffu, differs) : !__syncthreads_or(differs);
    const float cut = mean + a.alpha * sd;
    T* y = reinterpret_cast<T*>(a.y) + r * K;
#pragma unroll
    for (int i = 0; i < NCH; ++i) {
      const int c = (t + i * THREADS) * VEC;
      if (c < K) {
#pragma unroll
        for (int j = 0; j < VEC; ++j) v[i][j] = flat ? 0.f : fmaxf(v[i][j] - cut, 0.f);
        dsm_st<T, VEC>(y + c, v[i]);
      }
    }
  }
}

// Rows longer than DSM_CTA_MAX, a CTA per row: the sum, the centred sum of squares and the output are three passes over
// x; the first two load with the default policy so that the later ones can hit L2.
template <typename T, int VEC>
__global__ void __launch_bounds__(DSM_CTA_THREADS) sparse_relu_long_kernel(SreluArgs a) {
  __shared__ float sh[32];
  const int K = a.K;
  for (long long r = blockIdx.x; r < a.N; r += gridDim.x) {
    const T* x = reinterpret_cast<const T*>(a.x) + r * K;
    const float x0 = to_f32<T>(__ldg(x));
    float s = 0.f, q = 0.f;
    bool differs = false;
    for (int c = threadIdx.x * VEC; c < K; c += DSM_CTA_THREADS * VEC) {
      float v[VEC];
      dsm_ld<T, VEC, false>(x + c, v);
#pragma unroll
      for (int j = 0; j < VEC; ++j) { s += v[j]; differs |= v[j] != x0; }
    }
    const float mean = dsm_reduce<false>(s, DSM_CTA_THREADS, sh) / (float)K;
    for (int c = threadIdx.x * VEC; c < K; c += DSM_CTA_THREADS * VEC) {
      float v[VEC];
      dsm_ld<T, VEC, false>(x + c, v);
#pragma unroll
      for (int j = 0; j < VEC; ++j) { const float d = v[j] - mean; q += d * d; }
    }
    const float sd = sqrtf(dsm_reduce<false>(q, DSM_CTA_THREADS, sh) / (float)K);
    const bool flat = !__syncthreads_or(differs);
    const float cut = mean + a.alpha * sd;
    T* y = reinterpret_cast<T*>(a.y) + r * K;
    for (int c = threadIdx.x * VEC; c < K; c += DSM_CTA_THREADS * VEC) {
      float v[VEC];
      dsm_ld<T, VEC, true>(x + c, v);
#pragma unroll
      for (int j = 0; j < VEC; ++j) v[j] = flat ? 0.f : fmaxf(v[j] - cut, 0.f);
      dsm_st<T, VEC>(y + c, v);
    }
  }
}

template <typename T>
int launch_sparse_relu(const SreluArgs& a, bool vec, cudaStream_t s) {
  constexpr int V = 16 / sizeof(T);
  const char* name;
  if (a.K <= DSM_WARP_MAX) {
    constexpr int NV = DSM_WARP_MAX / 32 / V;
    const long long ctas = (a.N + DSM_WARPS - 1) / DSM_WARPS;
    const unsigned grid = (unsigned)(ctas < SRELU_MAX_CTAS ? ctas : SRELU_MAX_CTAS);
    if (vec) sparse_relu_kernel<T, V, NV, 32><<<grid, 32 * DSM_WARPS, 0, s>>>(a);
    else     sparse_relu_kernel<T, 1, 32, 32><<<grid, 32 * DSM_WARPS, 0, s>>>(a);
    name = "sparse_relu_warp";
  } else {
    const unsigned grid = (unsigned)(a.N < SRELU_MAX_CTAS ? a.N : SRELU_MAX_CTAS);
    if (a.K <= DSM_CTA_MAX) {
      constexpr int NV = DSM_CTA_MAX / DSM_CTA_THREADS / V, NS = DSM_CTA_MAX / DSM_CTA_THREADS;
      if (vec) sparse_relu_kernel<T, V, NV, DSM_CTA_THREADS><<<grid, DSM_CTA_THREADS, 0, s>>>(a);
      else     sparse_relu_kernel<T, 1, NS, DSM_CTA_THREADS><<<grid, DSM_CTA_THREADS, 0, s>>>(a);
      name = "sparse_relu_cta";
    } else {
      if (vec) sparse_relu_long_kernel<T, V><<<grid, DSM_CTA_THREADS, 0, s>>>(a);
      else     sparse_relu_long_kernel<T, 1><<<grid, DSM_CTA_THREADS, 0, s>>>(a);
      name = "sparse_relu_long";
    }
  }
  return check_launch(name);
}

// dx = y > 0 ? dy : +0, elementwise over n entries
template <typename T, int VEC>
__global__ void __launch_bounds__(EW_THREADS) relu_mask_grad_kernel(const T* dy, const T* y, T* dx, long long n) {
  const long long chunks = n / VEC;
  for (long long c = (long long)blockIdx.x * EW_THREADS + threadIdx.x; c < chunks; c += (long long)gridDim.x * EW_THREADS) {
    float d[VEC], w[VEC];
    dsm_ld<T, VEC, true>(dy + c * VEC, d);
    dsm_ld<T, VEC, true>(y + c * VEC, w);
#pragma unroll
    for (int j = 0; j < VEC; ++j) d[j] = w[j] > 0.f ? d[j] : 0.f;
    dsm_st<T, VEC>(dx + c * VEC, d);
  }
}

template <typename T>
int launch_relu_mask_grad(const void* dy, const void* y, void* dx, long long n, bool vec, cudaStream_t s) {
  constexpr int V = 16 / sizeof(T);
  const long long chunks = n / (vec ? V : 1), blocks = (chunks + EW_THREADS - 1) / EW_THREADS;
  const unsigned grid = (unsigned)(blocks < 65536 * 4 ? blocks : 65536 * 4);
  const T* d = reinterpret_cast<const T*>(dy);
  const T* w = reinterpret_cast<const T*>(y);
  if (vec) relu_mask_grad_kernel<T, V><<<grid, EW_THREADS, 0, s>>>(d, w, reinterpret_cast<T*>(dx), n);
  else     relu_mask_grad_kernel<T, 1><<<grid, EW_THREADS, 0, s>>>(d, w, reinterpret_cast<T*>(dx), n);
  return check_launch("relu_mask_grad");
}

}  // namespace bsmm
