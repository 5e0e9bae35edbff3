// Conv edge bias and channel-wise linear (bsmm_edge_bias, bsmm_edge_bias_grad, bsmm_cwise_linear,
// bsmm_cwise_linear_grad in include/bsmm_b200.h): the two per-channel ops of the reference's conv module.
//
// Both move bytes and compute almost nothing, so the element-wise passes are flat streams over the tensor: thread c owns
// the VEC elements at c * VEC (16-byte accesses when the pointers allow, one scalar chunk at the end), and walks the
// (outer, inner) coordinates of its elements from one division per chunk. Offsets are 64-bit; the division is 32-bit
// when the tensor has fewer than 2^32 elements.
//   * edge bias: the host builds pos_edge[p], the edge pattern of output position p or -1. y = x * g + b at edge
//     positions and x elsewhere, in one read of x and one write of y. Channels last: inner k, outer p, g / b [E][K];
//     channels first: inner p, outer k, g / b [K][E]. dx is the same pass with b absent.
//   * edge bias inference: in place, over the edge positions only, through the reference's table (int32 (offset, count)
//     per edge, then the positions of each edge).
//   * cwise_linear: inner = D*H*W, outer = C; y = a * x + b or a * (x + b), then relu.
//
// Reductions (dg / db of the edge bias, da / db of cwise_linear) go into fp32 partials over chunks that depend on the
// shape only; each partial is a fixed-order sum (in order per thread, then the xor-shuffle tree, then the warps in
// order). A last kernel adds the partials of each output in a fixed order: ln_reduce_partials_kernel (csrc/layer_norm.cuh)
// adds dg and db of the edge bias in one launch (their [parts][edges * K] layout is its), bias_grad_reduce_kernel
// (csrc/ewops.cuh) each sum cwise_linear returns. No atomics and no grid that depends on the SM count, so the gradients
// are bitwise reproducible.
//   * edge bias: the (n, j) pairs of edge e (n < N, j < count_e) in chunks of R; partial (s, f) sums chunk s of the
//     pairs of output f = (e, k). Channels last: one thread per (k, e, s); channels first: one warp.
//   * cwise_linear, D*H*W = 1: x is (N, C); thread (p, columns) adds rows [p * rp, (p + 1) * rp) of its VEC columns, as
//     bias_relu_grad does on its last axis (br_rows_per_part).
//   * cwise_linear, D*H*W > 1: CTA (s, c) adds elements [s * CW_SEG, +CW_SEG) of channel c's N * D*H*W elements in
//     16-byte chunks, chunk i * 256 + t to thread t, so each warp access is contiguous.
#pragma once
#include "ewops.cuh"
#include "layer_norm.cuh"

namespace bsmm {

constexpr int EB_BUDGET = 1 << 20;     // about this many (chunk, output) partials of dg / db at most
constexpr int EB_MIN_CHUNK = 32;       // (n, j) pairs per dg / db chunk, at least
constexpr int CW_SEG = 8192;           // cwise_linear, DHW > 1: elements of one channel per CTA and da / db partial

// coordinates of flat element i: inner = i % L_in, outer = (i / L_in) % L_out
__device__ __forceinline__ void flat_pos(long long i, long long L_in, long long L_out, bool narrow, long long& in,
                                         long long& out) {
  if (narrow) {
    const unsigned r = (unsigned)i / (unsigned)L_in;
    in = (unsigned)i - r * (unsigned)L_in;
    out = r % (unsigned)L_out;
  } else {
    const long long r = i / L_in;
    in = i - r * L_in;
    out = r % L_out;
  }
}

__device__ __forceinline__ void flat_next(long long& in, long long& out, long long L_in, long long L_out) {
  if (++in == L_in) {
    in = 0;
    if (++out == L_out) out = 0;
  }
}

template <typename T, int VEC>
__device__ __forceinline__ void flat_load(const T* p, long long i0, long long n, float (&v)[VEC]) {
  if (i0 + VEC <= n) {
    dsm_ld<T, VEC, true>(p + i0, v);
  } else {
#pragma unroll
    for (int j = 0; j < VEC; ++j) v[j] = i0 + j < n ? to_f32<T>(__ldcs(p + i0 + j)) : 0.f;
  }
}

template <typename T, int VEC>
__device__ __forceinline__ void flat_store(T* p, long long i0, long long n, const float (&v)[VEC]) {
  if (i0 + VEC <= n) {
    dsm_st<T, VEC>(p + i0, v);
  } else {
#pragma unroll
    for (int j = 0; j < VEC; ++j)
      if (i0 + j < n) __stcs(p + i0 + j, from_f32<T>(v[j]));
  }
}

// ---- edge bias ---------------------------------------------------------------------------------------------------------
struct EbArgs {
  const void* x;              // forward: x; gradient: dy
  const void* x2;             // gradient: x
  void* y;                    // forward: y (x itself for inference); gradient: dx
  const int32_t* pos_edge;    // [MPQ]
  const int32_t* lut;         // [2 E + entries]: (offset, count) per edge, then the positions
  const float* g;
  const float* b;             // NULL: y = x * g (the gradient's dx)
  float* part;
  long long n, N, MPQ, R;     // n = N * MPQ * K elements; R = (n, j) pairs per dg / db chunk
  int K, E, entries, S, layout;
};

template <typename T, int VEC>
__global__ void __launch_bounds__(EW_THREADS) edge_bias_kernel(EbArgs a) {
  const long long L_in = a.layout ? a.K : a.MPQ, L_out = a.layout ? a.MPQ : a.K;
  const long long chunks = (a.n + VEC - 1) / VEC;
  const bool narrow = a.n <= 0xffffffffLL;
  const T* x = static_cast<const T*>(a.x);
  T* y = static_cast<T*>(a.y);
  for (long long c = (long long)blockIdx.x * EW_THREADS + threadIdx.x; c < chunks; c += (long long)gridDim.x * EW_THREADS) {
    const long long i0 = c * VEC;
    long long in, out;
    flat_pos(i0, L_in, L_out, narrow, in, out);
    float v[VEC];
    flat_load<T, VEC>(x, i0, a.n, v);
    if (a.layout && a.K % VEC == 0) {      // the chunk's VEC channels share one position: one table read
      const int e = __ldg(a.pos_edge + out);
      if (e >= 0) {
        const long long gi = (long long)e * a.K + in;
#pragma unroll
        for (int j = 0; j < VEC; ++j)
          v[j] = a.b ? fmaf(v[j], __ldg(a.g + gi + j), __ldg(a.b + gi + j)) : v[j] * __ldg(a.g + gi + j);
      }
      flat_store<T, VEC>(y, i0, a.n, v);
      continue;
    }
    if (!a.layout && VEC > 1 && a.MPQ % VEC == 0) {   // one channel, VEC consecutive positions: 16-byte table reads
      int e[VEC];
#pragma unroll
      for (int j = 0; j < VEC; j += 4) {
        const int4 q = __ldg(reinterpret_cast<const int4*>(a.pos_edge + in + j));
        e[j] = q.x; e[j + 1] = q.y; e[j + 2] = q.z; e[j + 3] = q.w;
      }
#pragma unroll
      for (int j = 0; j < VEC; ++j) {
        if (e[j] >= 0) {
          const long long gi = out * a.E + e[j];
          v[j] = a.b ? fmaf(v[j], __ldg(a.g + gi), __ldg(a.b + gi)) : v[j] * __ldg(a.g + gi);
        }
      }
      flat_store<T, VEC>(y, i0, a.n, v);
      continue;
    }
#pragma unroll
    for (int j = 0; j < VEC; ++j) {
      const long long p = a.layout ? out : in, k = a.layout ? in : out;
      const int e = __ldg(a.pos_edge + p);
      if (e >= 0) {
        const long long gi = a.layout ? (long long)e * a.K + k : k * a.E + e;
        v[j] = a.b ? fmaf(v[j], __ldg(a.g + gi), __ldg(a.b + gi)) : v[j] * __ldg(a.g + gi);
      }
      flat_next(in, out, L_in, L_out);
    }
    flat_store<T, VEC>(y, i0, a.n, v);
  }
}

// q = a / b, r = a % b, in 32 bits when the operands fit
__device__ __forceinline__ void udivmod(long long a, long long b, bool narrow, long long& q, long long& r) {
  if (narrow) {
    const unsigned qq = (unsigned)a / (unsigned)b;
    q = qq;
    r = (unsigned)a - qq * (unsigned)b;
  } else {
    q = a / b;
    r = a - q * b;
  }
}

// In place over the N * entries * K edge elements: channels last in (n, j, k) order, VEC channels per thread;
// channels first in (n, k, j) order, one element per thread. The edge of entry j is found in the table's header.
template <typename T, int VEC>
__global__ void __launch_bounds__(EW_THREADS) edge_bias_inference_kernel(EbArgs a) {
  const long long KV = a.layout ? a.K / VEC : 1, total = a.N * a.entries * (a.layout ? KV : a.K);
  const bool narrow = total <= 0xffffffffLL;
  T* y = static_cast<T*>(a.y);
  for (long long t = (long long)blockIdx.x * EW_THREADS + threadIdx.x; t < total; t += (long long)gridDim.x * EW_THREADS) {
    long long j, k, n, r;
    if (a.layout) {
      udivmod(t, KV, narrow, r, k);
      k *= VEC;
      udivmod(r, a.entries, narrow, n, j);
    } else {
      udivmod(t, a.entries, narrow, r, j);
      udivmod(r, a.K, narrow, n, k);
    }
    // the last edge whose first entry is at or before entry j (the data follow the 2 E header words)
    const int jj = 2 * a.E + (int)j;
    int lo = 0, hi = a.E - 1;
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (__ldg(a.lut + 2 * mid) <= jj) lo = mid; else hi = mid - 1;
    }
    const long long p = __ldg(a.lut + jj);
    const long long off = a.layout ? (n * a.MPQ + p) * a.K + k : (n * a.K + k) * a.MPQ + p;
    const long long gi = a.layout ? (long long)lo * a.K + k : k * a.E + lo;
    float v[VEC];
    dsm_ld<T, VEC, false>(y + off, v);
#pragma unroll
    for (int i = 0; i < VEC; ++i) v[i] = fmaf(v[i], __ldg(a.g + gi + i), __ldg(a.b + gi + i));
    dsm_st<T, VEC>(y + off, v);
  }
}

// Partials of dg and db, channels last: thread (k, e, s) adds chunk s of edge e's (n, j) pairs in order.
template <typename T>
__global__ void __launch_bounds__(128) edge_bias_grad_nhwc_kernel(EbArgs a) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x, e = blockIdx.y, s = blockIdx.z;
  if (k >= a.K) return;
  const int off = __ldg(a.lut + 2 * e), cnt = __ldg(a.lut + 2 * e + 1);
  const T* dy = static_cast<const T*>(a.x);
  const T* x = static_cast<const T*>(a.x2);
  const long long t0 = s * a.R, t1 = min(a.N * cnt, t0 + a.R);
  float dg = 0.f, db = 0.f;
  if (t0 < t1) {
    long long n = t0 / cnt;
    int j = (int)(t0 - n * cnt);
#pragma unroll 4
    for (long long t = t0; t < t1; ++t) {
      const long long o = (n * a.MPQ + __ldg(a.lut + off + j)) * a.K + k;
      const float d = to_f32<T>(__ldcs(dy + o));
      dg = fmaf(d, to_f32<T>(__ldcs(x + o)), dg);
      db += d;
      if (++j == cnt) { j = 0; ++n; }
    }
  }
  const long long F = (long long)a.E * a.K, f = (long long)e * a.K + k;
  a.part[s * F + f] = dg;
  a.part[(a.S + s) * F + f] = db;
}

// Partials of dg and db, channels first: warp (k, e, s) adds chunk s of edge e's (n, j) pairs, lane l the pairs
// l, l + 32, ... in order, then the xor-shuffle tree.
template <typename T>
__global__ void __launch_bounds__(256) edge_bias_grad_nchw_kernel(EbArgs a) {
  const int lane = threadIdx.x & 31, k = blockIdx.x * 8 + (threadIdx.x >> 5), e = blockIdx.y, s = blockIdx.z;
  if (k >= a.K) return;
  const int off = __ldg(a.lut + 2 * e), cnt = __ldg(a.lut + 2 * e + 1);
  const T* dy = static_cast<const T*>(a.x);
  const T* x = static_cast<const T*>(a.x2);
  const long long t1 = min(a.N * cnt, (s + 1) * a.R);
  float dg = 0.f, db = 0.f;
  for (long long t = s * a.R + lane; t < t1; t += 32) {
    const long long n = t / cnt;
    const long long o = (n * a.K + k) * a.MPQ + __ldg(a.lut + off + (int)(t - n * cnt));
    const float d = to_f32<T>(__ldcs(dy + o));
    dg = fmaf(d, to_f32<T>(__ldcs(x + o)), dg);
    db += d;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    dg += __shfl_xor_sync(0xffffffffu, dg, o);
    db += __shfl_xor_sync(0xffffffffu, db, o);
  }
  if (lane == 0) {
    const long long F = (long long)a.E * a.K, f = (long long)k * a.E + e;
    a.part[s * F + f] = dg;
    a.part[(a.S + s) * F + f] = db;
  }
}

// (R, S) of the dg / db partition: chunks of R pairs of the longest edge's N * max_count, about EB_BUDGET partials in
// all and at most 65535 chunks (grid.z).
inline void eb_chunks(long long N, int max_count, long long F, long long& R, int& S) {
  const long long work = N * max_count;
  long long target = EB_BUDGET / (F > 0 ? F : 1);
  target = target < 1 ? 1 : (target > 65535 ? 65535 : target);
  R = (work + target - 1) / target;
  if (R < EB_MIN_CHUNK) R = EB_MIN_CHUNK;
  S = (int)((work + R - 1) / R);
}

inline unsigned flat_grid(long long chunks) {
  const long long g = (chunks + EW_THREADS - 1) / EW_THREADS;
  return (unsigned)(g < (1LL << 20) ? (g > 0 ? g : 1) : (1LL << 20));
}

template <typename T>
int launch_edge_bias(EbArgs& a, bool vec, const char* name, cudaStream_t s) {
  constexpr int V = 16 / sizeof(T);
  if (vec) edge_bias_kernel<T, V><<<flat_grid((a.n + V - 1) / V), EW_THREADS, 0, s>>>(a);
  else     edge_bias_kernel<T, 1><<<flat_grid(a.n), EW_THREADS, 0, s>>>(a);
  return check_launch(name);
}

template <typename T>
int launch_edge_bias_inference(EbArgs& a, bool vec, cudaStream_t s) {
  constexpr int V = 16 / sizeof(T);
  if (vec && a.layout) edge_bias_inference_kernel<T, V><<<flat_grid(a.N * a.entries * (a.K / V)), EW_THREADS, 0, s>>>(a);
  else                 edge_bias_inference_kernel<T, 1><<<flat_grid(a.N * a.entries * a.K), EW_THREADS, 0, s>>>(a);
  return check_launch("edge_bias_inference");
}

template <typename T>
int launch_edge_bias_grad(EbArgs& a, bool vec, float* dg, float* db, cudaStream_t s) {
  if (a.n > 0) {
    if (int e = launch_edge_bias<T>(a, vec, "edge_bias_grad", s)) return e;
    if (a.S > 0) {
      if (a.layout) {
        const int threads = a.K <= 32 ? 32 : (a.K <= 64 ? 64 : 128);
        const dim3 grid((unsigned)((a.K + threads - 1) / threads), (unsigned)a.E, (unsigned)a.S);
        edge_bias_grad_nhwc_kernel<T><<<grid, threads, 0, s>>>(a);
      } else {
        const dim3 grid((unsigned)((a.K + 7) / 8), (unsigned)a.E, (unsigned)a.S);
        edge_bias_grad_nchw_kernel<T><<<grid, 256, 0, s>>>(a);
      }
      if (int e = check_launch("edge_bias_grad")) return e;
    }
  }
  const int F = a.E * a.K;
  ln_reduce_partials_kernel<float><<<(unsigned)((F + 255) / 256), 256, 0, s>>>(a.part, a.S, F, dg, db);
  return check_launch("edge_bias_grad");
}

// ---- cwise_linear ------------------------------------------------------------------------------------------------------
struct CwArgs {
  const void* x;     // forward: x; gradient: dy
  const void* src;   // gradient: x with a gain, y for relu without one, else unused
  void* y;           // forward: y; gradient: dx (unused without gain and relu)
  const float* a;    // NULL: no gain
  const float* b;    // NULL: no bias
  float* part;
  long long n, N, DHW, rp, parts;
  int C, relu, swap, want_a, want_b;
};

// the forward's fp32 expression, which the gradient's relu mask reuses
__device__ __forceinline__ float cw_fwd(float x, float a, float b, bool has_b, int swap) {
  if (!has_b) return a * x;
  return swap ? a * (x + b) : fmaf(a, x, b);
}

template <typename T, int VEC>
__global__ void __launch_bounds__(EW_THREADS) cwise_linear_kernel(CwArgs a) {
  const long long chunks = (a.n + VEC - 1) / VEC;
  const bool narrow = a.n <= 0xffffffffLL, has_b = a.b != nullptr;
  const T* x = static_cast<const T*>(a.x);
  T* y = static_cast<T*>(a.y);
  for (long long c = (long long)blockIdx.x * EW_THREADS + threadIdx.x; c < chunks; c += (long long)gridDim.x * EW_THREADS) {
    const long long i0 = c * VEC;
    long long p, ch;
    flat_pos(i0, a.DHW, a.C, narrow, p, ch);
    float v[VEC];
    flat_load<T, VEC>(x, i0, a.n, v);
#pragma unroll
    for (int j = 0; j < VEC; ++j) {
      const float g = a.a ? __ldg(a.a + ch) : 1.f, b = has_b ? __ldg(a.b + ch) : 0.f;
      const float z = cw_fwd(v[j], g, b, has_b, a.swap);
      v[j] = a.relu ? fmaxf(z, 0.f) : z;
      flat_next(p, ch, a.DHW, a.C);
    }
    flat_store<T, VEC>(y, i0, a.n, v);
  }
}

// one element of the gradient: dx, and the terms of da and db
__device__ __forceinline__ void cw_bwd(const CwArgs& A, float dy, float s, float g, float b, float& dx, float& ta,
                                       float& tb) {
  if (A.a) {
    const float z = cw_fwd(s, g, b, A.b != nullptr, A.swap);
    const float d = A.relu && !(z > 0.f) ? 0.f : dy;
    dx = d * g;
    ta = A.swap ? d * (s + b) : d * s;
    tb = A.swap ? dx : d;
  } else {
    dx = A.relu && !(s > 0.f) ? 0.f : dy;
    ta = 0.f;
    tb = dx;
  }
}

// D*H*W = 1: x (N, C); thread (p, columns [c0, c0 + VEC)) over rows [p * rp, (p + 1) * rp)
template <typename T, int VEC>
__global__ void __launch_bounds__(EW_THREADS) cwise_linear_grad_nc_kernel(CwArgs a, int tpr) {
  const int CV = a.C / VEC, cv = blockIdx.x * tpr + threadIdx.x % tpr;
  if (cv >= CV) return;
  const int c0 = cv * VEC, rpc = EW_THREADS / tpr;
  const bool rd = a.a || a.relu;
  float gv[VEC], bv[VEC];
#pragma unroll
  for (int j = 0; j < VEC; ++j) {
    gv[j] = a.a ? __ldg(a.a + c0 + j) : 1.f;
    bv[j] = a.b ? __ldg(a.b + c0 + j) : 0.f;
  }
  for (long long p = (long long)blockIdx.y * rpc + threadIdx.x / tpr; p < a.parts; p += (long long)gridDim.y * rpc) {
    float sa[VEC], sb[VEC];
#pragma unroll
    for (int j = 0; j < VEC; ++j) sa[j] = sb[j] = 0.f;
    const long long r1 = min(a.N, (p + 1) * a.rp);
#pragma unroll 4
    for (long long r = p * a.rp; r < r1; ++r) {
      const long long off = r * a.C + c0;
      float d[VEC], s[VEC];
      dsm_ld<T, VEC, true>(static_cast<const T*>(a.x) + off, d);
      if (rd) dsm_ld<T, VEC, true>(static_cast<const T*>(a.src) + off, s);
#pragma unroll
      for (int j = 0; j < VEC; ++j) {
        float ta, tb;
        cw_bwd(a, d[j], rd ? s[j] : 0.f, gv[j], bv[j], d[j], ta, tb);
        sa[j] += ta;
        sb[j] += tb;
      }
      if (rd) dsm_st<T, VEC>(static_cast<T*>(a.y) + off, d);
    }
#pragma unroll
    for (int j = 0; j < VEC; ++j) {
      if (a.want_a) a.part[p * a.C + c0 + j] = sa[j];
      if (a.want_b) a.part[(a.parts + p) * a.C + c0 + j] = sb[j];
    }
  }
}

// D*H*W > 1: CTA (s, c) over elements [s * CW_SEG, +CW_SEG) of channel c's N * DHW, in chunks of V = 16 / sizeof(T)
// elements: thread t adds, in order, chunks i * EW_THREADS + t for i < CW_SEG / (EW_THREADS * V), so a warp's 16-byte
// accesses are contiguous. On the scalar route (VEC = 1) a thread reads the same chunks element by element, so the
// elements each thread adds, and their order, do not depend on the access width.
template <typename T, int VEC>
__global__ void __launch_bounds__(EW_THREADS) cwise_linear_grad_seg_kernel(CwArgs a) {
  constexpr int V = 16 / sizeof(T), CHUNKS = CW_SEG / (EW_THREADS * V);
  static_assert(VEC == 1 || VEC == V, "16-byte chunks or single elements");
  __shared__ float red[2][EW_THREADS / 32];
  const long long ND = a.N * a.DHW, base = (long long)blockIdx.x * CW_SEG + threadIdx.x * V;
  const bool rd = a.a || a.relu, narrow = ND <= 0xffffffffLL;
  // dx never overlaps dy or x: restrict lets the loads of later chunks start before the stores of earlier ones
  const T* __restrict__ dy = static_cast<const T*>(a.x);
  const T* __restrict__ src = static_cast<const T*>(a.src);
  T* __restrict__ dx = static_cast<T*>(a.y);
  for (long long c = blockIdx.y; c < a.C; c += gridDim.y) {
    const float g = a.a ? __ldg(a.a + c) : 1.f, b = a.b ? __ldg(a.b + c) : 0.f;
    float sa = 0.f, sb = 0.f;
#pragma unroll
    for (int i = 0; i < CHUNKS; ++i) {
      const long long t0 = base + (long long)i * EW_THREADS * V;
      if (t0 < ND) {
        long long n, p;
        udivmod(t0, a.DHW, narrow, n, p);
#pragma unroll
        for (int q = 0; q < V; q += VEC) {
          if (t0 + q < ND) {     // on the vector route DHW % V == 0: a chunk is all in or all out
            const long long off = (n * a.C + c) * a.DHW + p;
            float d[VEC], v[VEC];
            dsm_ld<T, VEC, true>(dy + off, d);
            if (rd) dsm_ld<T, VEC, true>(src + off, v);
#pragma unroll
            for (int j = 0; j < VEC; ++j) {
              float ta, tb;
              cw_bwd(a, d[j], rd ? v[j] : 0.f, g, b, d[j], ta, tb);
              sa += ta;
              sb += tb;
            }
            if (rd) dsm_st<T, VEC>(dx + off, d);
          }
          p += VEC;
          if (p >= a.DHW) { p -= a.DHW; ++n; }
        }
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      sa += __shfl_xor_sync(0xffffffffu, sa, o);
      sb += __shfl_xor_sync(0xffffffffu, sb, o);
    }
    if ((threadIdx.x & 31) == 0) { red[0][threadIdx.x >> 5] = sa; red[1][threadIdx.x >> 5] = sb; }
    __syncthreads();
    if (threadIdx.x == 0) {
      float ta = 0.f, tb = 0.f;
#pragma unroll
      for (int w = 0; w < EW_THREADS / 32; ++w) { ta += red[0][w]; tb += red[1][w]; }
      if (a.want_a) a.part[blockIdx.x * a.C + c] = ta;
      if (a.want_b) a.part[(a.parts + blockIdx.x) * a.C + c] = tb;
    }
    __syncthreads();
  }
}

inline long long cw_rows_per_part(long long N, int C) { return br_rows_per_part(N, C); }

inline long long cw_parts(long long N, int C, long long DHW) {
  if (DHW == 1) return (N + cw_rows_per_part(N, C) - 1) / cw_rows_per_part(N, C);
  return (N * DHW + CW_SEG - 1) / CW_SEG;
}

template <typename T>
int launch_cwise_linear(CwArgs& a, bool vec, cudaStream_t s) {
  constexpr int V = 16 / sizeof(T);
  if (vec) cwise_linear_kernel<T, V><<<flat_grid((a.n + V - 1) / V), EW_THREADS, 0, s>>>(a);
  else     cwise_linear_kernel<T, 1><<<flat_grid(a.n), EW_THREADS, 0, s>>>(a);
  return check_launch("cwise_linear");
}

template <typename T, int VEC>
void cw_grad_launch(CwArgs& a, cudaStream_t s) {
  if (a.DHW == 1) {
    const int CV = a.C / VEC;
    int tpr = 1;
    while (tpr < CV && tpr < EW_THREADS) tpr *= 2;
    const long long rpc = EW_THREADS / tpr, gy = (a.parts + rpc - 1) / rpc;
    const dim3 grid((unsigned)((CV + tpr - 1) / tpr), (unsigned)(gy < 65535 ? gy : 65535));
    cwise_linear_grad_nc_kernel<T, VEC><<<grid, EW_THREADS, 0, s>>>(a, tpr);
  } else {
    const dim3 grid((unsigned)a.parts, (unsigned)(a.C < 65535 ? a.C : 65535));
    cwise_linear_grad_seg_kernel<T, VEC><<<grid, EW_THREADS, 0, s>>>(a);
  }
}

template <typename T>
int launch_cwise_linear_grad(CwArgs& a, bool vec, float* da, float* db, cudaStream_t s) {
  constexpr int V = 16 / sizeof(T);
  const char* name = a.DHW == 1 ? "cwise_linear_grad_nc" : "cwise_linear_grad_ncdhw";
  if (a.n > 0) {
    if (vec) cw_grad_launch<T, V>(a, s);
    else     cw_grad_launch<T, 1>(a, s);
    if (int e = check_launch(name)) return e;
  }
  const unsigned rg = (unsigned)((a.C + 7) / 8);
  if (da) bias_grad_reduce_kernel<float><<<rg, 256, 0, s>>>(a.part, a.parts, 1, a.C, a.C, da);
  if (db) bias_grad_reduce_kernel<float><<<rg, 256, 0, s>>>(a.part + a.parts * a.C, a.parts, 1, a.C, a.C, db);
  return check_launch(name);
}

}  // namespace bsmm
