// LSTM gate nonlinearity and sparse relu (bsmm_lstm_gates, bsmm_lstm_gates_grad, bsmm_sparse_relu, bsmm_relu_mask_grad
// in include/bsmm_b200.h).
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
