// Bias + activation and dropout (bsmm_bias_relu, bsmm_bias_relu_grad, bsmm_dropout_mask, bsmm_dropout_apply in
// include/bsmm_b200.h).
//
// bias_relu: y = act(x + b) along the feature axis, in fp32 with one final rounding. These ops move bytes and compute
// almost nothing, so the kernels stream x once and y once, with 16-byte accesses where every row start allows.
//   * feature axis last, x (N, K): thread (p, c) owns the VEC columns at c * VEC and the rows of partial p,
//     [p * rp, (p + 1) * rp), which it walks in order; the gradient adds its dx values in that order and stores one fp32
//     partial of db per (p, column).
//   * feature axis 0, x (K, N): CTA (s, k) owns elements [s * BR_SEG, +BR_SEG) of row k, thread t the 8 contiguous ones
//     at t * 8; the gradient adds them in order, then the xor-shuffle tree, then the warps in order: one partial per
//     (k, s).
// A last kernel adds the partials of each feature in a fixed order. rp and BR_SEG depend on the shape only, and the
// per-element order does not depend on the access width, so db is bitwise reproducible without atomics.
//
// dropout: the reference's mask format (bit e % 32 of word e / 32 set = keep element e) drawn from counter-based
// Philox4x32-10: key = the 64-bit seed, counter = (e / 4 as 64 bits, call as 64 bits), output word e % 4, keep iff that
// word < floor(keep_prob * 2^32), compared in 64 bits. seed and call live in device memory ([seed, call], int64); the
// mask kernel reads them there and a one-thread kernel after it advances call, so a mask depends on (seed, call, M) only
// and every replay of a captured graph draws a new one.
#pragma once
#include "dense_softmax.cuh"
#include "philox.cuh"

namespace bsmm {

enum { ACT_NONE = 0, ACT_RELU = 1, ACT_FAST_GELU = 2 };
constexpr int EW_THREADS = 256;
constexpr int BR_SEG = 8 * EW_THREADS;   // axis 0: elements of one row per CTA and per db partial
constexpr float GELU_A = 1.702f;         // fast_gelu(z) = z * sigmoid(1.702 z), the reference's ew_swish(z, 1.702)
constexpr int DROP_MAX_DIMS = 8;

struct BrArgs {
  const void* x;     // forward: x; gradient: dy
  const void* src;   // gradient: y (relu) or x (fast_gelu)
  const void* b;
  void* y;           // forward: y; gradient: dx (not written without an activation)
  float* part;       // gradient: fp32 partials of db
  long long N, rp, parts;
  int K, bdt, act;
};

__device__ __forceinline__ float ew_param(const void* p, int dt, long long i) {
  if (dt == BSMM_F32) return __ldg(reinterpret_cast<const float*>(p) + i);
  if (dt == BSMM_F16) return __half2float(__ldg(reinterpret_cast<const __half*>(p) + i));
  return __bfloat162float(__ldg(reinterpret_cast<const __nv_bfloat16*>(p) + i));
}

__device__ __forceinline__ float br_sigmoid(float z) { return 1.f / (1.f + expf(-GELU_A * z)); }

__device__ __forceinline__ float br_fwd(float z, int act) {
  if (act == ACT_RELU) return fmaxf(z, 0.f);
  if (act == ACT_FAST_GELU) return z * br_sigmoid(z);
  return z;
}

// dx of one element: relu reads y, fast_gelu reads x and recomputes z = x + b (reference ew_op_gpu.cu:1043-1070)
__device__ __forceinline__ float br_bwd(float dy, float s, float b, int act) {
  if (act == ACT_RELU) return s > 0.f ? dy : 0.f;
  if (act == ACT_FAST_GELU) {
    const float z = s + b, sg = br_sigmoid(z);
    return dy * (sg + GELU_A * z * sg * (1.f - sg));
  }
  return dy;
}

template <typename T, int VEC, bool GRAD>
__global__ void __launch_bounds__(EW_THREADS) bias_act_nc_kernel(BrArgs a, int tpr) {
  const int KV = a.K / VEC, cv = blockIdx.x * tpr + threadIdx.x % tpr;
  if (cv >= KV) return;
  const int k0 = cv * VEC, rpc = EW_THREADS / tpr;
  float bv[VEC];
#pragma unroll
  for (int j = 0; j < VEC; ++j) bv[j] = ew_param(a.b, a.bdt, k0 + j);
  for (long long p = (long long)blockIdx.y * rpc + threadIdx.x / tpr; p < a.parts; p += (long long)gridDim.y * rpc) {
    float s[VEC];
#pragma unroll
    for (int j = 0; j < VEC; ++j) s[j] = 0.f;
    const long long r1 = min(a.N, (p + 1) * a.rp);
#pragma unroll 4
    for (long long r = p * a.rp; r < r1; ++r) {
      const long long off = r * a.K + k0;
      float v[VEC];
      dsm_ld<T, VEC, true>(reinterpret_cast<const T*>(a.x) + off, v);
      if constexpr (!GRAD) {
#pragma unroll
        for (int j = 0; j < VEC; ++j) v[j] = br_fwd(v[j] + bv[j], a.act);
        dsm_st<T, VEC>(reinterpret_cast<T*>(a.y) + off, v);
      } else {
        if (a.act != ACT_NONE) {
          float w[VEC];
          dsm_ld<T, VEC, true>(reinterpret_cast<const T*>(a.src) + off, w);
#pragma unroll
          for (int j = 0; j < VEC; ++j) v[j] = br_bwd(v[j], w[j], bv[j], a.act);
          dsm_st<T, VEC>(reinterpret_cast<T*>(a.y) + off, v);
        }
#pragma unroll
        for (int j = 0; j < VEC; ++j) s[j] += v[j];
      }
    }
    if constexpr (GRAD) {
#pragma unroll
      for (int j = 0; j < VEC; ++j) a.part[p * a.K + k0 + j] = s[j];
    }
  }
}

template <typename T, int VEC, bool GRAD>
__global__ void __launch_bounds__(EW_THREADS) bias_act_cn_kernel(BrArgs a) {
  __shared__ float red[EW_THREADS / 32];
  const long long n0 = (long long)blockIdx.x * BR_SEG + threadIdx.x * 8;
  for (long long k = blockIdx.y; k < a.K; k += gridDim.y) {
    const float bk = ew_param(a.b, a.bdt, k);
    float s = 0.f;
#pragma unroll
    for (int c = 0; c < 8; c += VEC) {
      const long long n = n0 + c;
      if (n < a.N) {                      // on the vector route N % VEC == 0: a chunk is all in or all out
        const long long off = k * a.N + n;
        float v[VEC];
        dsm_ld<T, VEC, true>(reinterpret_cast<const T*>(a.x) + off, v);
        if constexpr (!GRAD) {
#pragma unroll
          for (int j = 0; j < VEC; ++j) v[j] = br_fwd(v[j] + bk, a.act);
          dsm_st<T, VEC>(reinterpret_cast<T*>(a.y) + off, v);
        } else {
          if (a.act != ACT_NONE) {
            float w[VEC];
            dsm_ld<T, VEC, true>(reinterpret_cast<const T*>(a.src) + off, w);
#pragma unroll
            for (int j = 0; j < VEC; ++j) v[j] = br_bwd(v[j], w[j], bk, a.act);
            dsm_st<T, VEC>(reinterpret_cast<T*>(a.y) + off, v);
          }
#pragma unroll
          for (int j = 0; j < VEC; ++j) s += v[j];
        }
      }
    }
    if constexpr (GRAD) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
      __syncthreads();
      if (threadIdx.x == 0) {
        float t = 0.f;
#pragma unroll
        for (int w = 0; w < EW_THREADS / 32; ++w) t += red[w];
        a.part[k * gridDim.x + blockIdx.x] = t;
      }
      __syncthreads();
    }
  }
}

// db[k] = sum over s of part[k * ks + s * ss]: warp w of the CTA owns feature k, lane l adds s = l, l + 32, ... in
// order, then the xor-shuffle tree; converted to G, the dtype of b.
template <typename G>
__global__ void __launch_bounds__(256) bias_grad_reduce_kernel(const float* part, long long S, long long ks, long long ss,
                                                               int K, void* db) {
  const long long k = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (k >= K) return;
  float t = 0.f;
  for (long long s = threadIdx.x & 31; s < S; s += 32) t += part[k * ks + s * ss];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
  if ((threadIdx.x & 31) == 0) reinterpret_cast<G*>(db)[k] = from_f32<G>(t);
}

// axis last: rows per db partial, about 2^20 (partial, feature) pairs and at least 8 rows each
inline long long br_rows_per_part(long long N, int K) {
  const long long rp = (N * K + (1LL << 20) - 1) >> 20;
  return rp < 8 ? 8 : rp;
}

inline long long br_parts(int axis, long long N, int K) {
  return axis == 0 ? (N + BR_SEG - 1) / BR_SEG : (N + br_rows_per_part(N, K) - 1) / br_rows_per_part(N, K);
}

inline size_t br_workspace_floats(int axis, long long N, int K) { return (size_t)br_parts(axis, N, K) * K; }

template <typename T, int VEC, bool GRAD>
void br_launch(BrArgs& a, int axis, cudaStream_t s) {
  if (axis == 0) {
    const dim3 grid((unsigned)a.parts, (unsigned)(a.K < 65535 ? a.K : 65535));
    bias_act_cn_kernel<T, VEC, GRAD><<<grid, EW_THREADS, 0, s>>>(a);
  } else {
    const int KV = a.K / VEC;
    int tpr = 1;
    while (tpr < KV && tpr < EW_THREADS) tpr *= 2;
    const long long rpc = EW_THREADS / tpr, gy = (a.parts + rpc - 1) / rpc;
    const dim3 grid((unsigned)((KV + tpr - 1) / tpr), (unsigned)(gy < 65535 ? gy : 65535));
    bias_act_nc_kernel<T, VEC, GRAD><<<grid, EW_THREADS, 0, s>>>(a, tpr);
  }
}

template <typename T>
int launch_bias_act(BrArgs& a, int axis, bool grad, bool vec, void* db, cudaStream_t s) {
  constexpr int V = 16 / sizeof(T);
  a.rp = br_rows_per_part(a.N, a.K);
  a.parts = br_parts(axis, a.N, a.K);
  if (grad) {
    if (vec) br_launch<T, V, true>(a, axis, s);
    else     br_launch<T, 1, true>(a, axis, s);
  } else {
    if (vec) br_launch<T, V, false>(a, axis, s);
    else     br_launch<T, 1, false>(a, axis, s);
  }
  const char* name = grad ? (axis ? "bias_relu_grad_nc" : "bias_relu_grad_cn") : (axis ? "bias_relu_nc" : "bias_relu_cn");
  if (!grad) return check_launch(name);
  if (int e = check_launch(name)) return e;
  const long long ks = axis ? 1 : a.parts, ss = axis ? a.K : 1;
  BSMM_DISPATCH_DTYPE(a.bdt, G, {
    bias_grad_reduce_kernel<G><<<(unsigned)((a.K + 7) / 8), 256, 0, s>>>(a.part, a.parts, ks, ss, a.K, db);
  });
  return check_launch(name);
}

// ---- dropout (philox4x32_10: philox.cuh) -----------------------------------------------------------------------------
// one thread per mask word: 8 Philox blocks of 4 elements; bits at or past M stay 0
__global__ void __launch_bounds__(EW_THREADS) dropout_mask_kernel(uint32_t* mask, long long M, unsigned long long thr,
                                                                  const long long* state) {
  const unsigned long long seed = (unsigned long long)state[0], call = (unsigned long long)state[1];
  const uint2 key = make_uint2((unsigned)seed, (unsigned)(seed >> 32));
  const long long words = (M + 31) / 32;
  for (long long w = (long long)blockIdx.x * EW_THREADS + threadIdx.x; w < words; w += (long long)gridDim.x * EW_THREADS) {
    uint32_t bits = 0;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const unsigned long long g = (unsigned long long)w * 8 + j;
      const uint4 r = philox4x32_10(make_uint4((unsigned)g, (unsigned)(g >> 32), (unsigned)call, (unsigned)(call >> 32)), key);
      const long long e = (long long)g * 4;
      bits |= (uint32_t)(e + 0 < M && r.x < thr) << (4 * j + 0);
      bits |= (uint32_t)(e + 1 < M && r.y < thr) << (4 * j + 1);
      bits |= (uint32_t)(e + 2 < M && r.z < thr) << (4 * j + 2);
      bits |= (uint32_t)(e + 3 < M && r.w < thr) << (4 * j + 3);
    }
    mask[w] = bits;
  }
}

__global__ void dropout_advance_kernel(long long* state) { state[1] += 1; }

inline int launch_dropout_mask(uint32_t* mask, long long M, unsigned long long thr, long long* state, cudaStream_t s) {
  const long long words = (M + 31) / 32, blocks = (words + EW_THREADS - 1) / EW_THREADS;
  dropout_mask_kernel<<<(unsigned)(blocks < 65536 ? blocks : 65536), EW_THREADS, 0, s>>>(mask, M, thr, state);
  if (int e = check_launch("dropout_mask")) return e;
  dropout_advance_kernel<<<1, 1, 0, s>>>(state);
  return check_launch("dropout_mask");
}

// x's dims after dropping size-1 dims and merging neighbours that index the mask alike; nd == 0 when the mask index of
// element e is e itself. Mask strides are 0 on broadcast dims; the innermost one is 0 or 1.
struct DropArgs {
  const void* x;
  const uint32_t* mask;
  void* y;
  long long n, words;
  long long size[DROP_MAX_DIMS], mst[DROP_MAX_DIMS];
  int nd;
  float scale;
};

__device__ __forceinline__ long long drop_divmod(long long& rem, long long size) {
  if (((unsigned long long)rem | (unsigned long long)size) >> 32 == 0) {
    const unsigned r = (unsigned)rem, d = (unsigned)size;
    rem = r / d;
    return r % d;
  }
  const long long i = rem % size;
  rem /= size;
  return i;
}

template <typename T, int VEC>
__global__ void __launch_bounds__(EW_THREADS) dropout_apply_kernel(DropArgs a) {
  const long long chunks = a.n / VEC;
  for (long long c = (long long)blockIdx.x * EW_THREADS + threadIdx.x; c < chunks; c += (long long)gridDim.x * EW_THREADS) {
    const long long e = c * VEC;
    long long m = 0;
    bool inner_bcast = false;
    if (a.nd == 0) {
      m = e;
    } else {
      long long rem = e;
      for (int d = a.nd - 1; d >= 0; --d) m += drop_divmod(rem, a.size[d]) * a.mst[d];
      inner_bcast = a.mst[a.nd - 1] == 0;
    }
    const long long w = m >> 5;
    unsigned long long bits = __ldg(reinterpret_cast<const unsigned*>(a.mask) + w);
    if (VEC > 1 && !inner_bcast && w + 1 < a.words)
      bits |= (unsigned long long)__ldg(reinterpret_cast<const unsigned*>(a.mask) + w + 1) << 32;
    bits >>= (m & 31);
    float v[VEC];
    dsm_ld<T, VEC, true>(reinterpret_cast<const T*>(a.x) + e, v);
#pragma unroll
    for (int j = 0; j < VEC; ++j) v[j] = (bits >> (inner_bcast ? 0 : j)) & 1 ? v[j] * a.scale : 0.f;
    dsm_st<T, VEC>(reinterpret_cast<T*>(a.y) + e, v);
  }
}

template <typename T>
int launch_dropout_apply(const DropArgs& a, bool vec, cudaStream_t s) {
  constexpr int V = 16 / sizeof(T);
  const long long chunks = a.n / (vec ? V : 1), blocks = (chunks + EW_THREADS - 1) / EW_THREADS;
  const unsigned grid = (unsigned)(blocks < 65536 * 4 ? blocks : 65536 * 4);
  if (vec) dropout_apply_kernel<T, V><<<grid, EW_THREADS, 0, s>>>(a);
  else     dropout_apply_kernel<T, 1><<<grid, EW_THREADS, 0, s>>>(a);
  return check_launch("dropout_apply");
}

}  // namespace bsmm
