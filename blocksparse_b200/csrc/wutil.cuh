// Utilities on the block-sparse weight format (blocks, bs, bs) and its neighbours on the hot path.
// All of them are HBM-bound passes over W (or over the activations), so the kernels are built around wide coalesced
// accesses and warp-shuffle reductions, one warp (or one small CTA) per block / block column, no atomics.
//
//   block_norm_kernel        per-block max|w| or l2 norm           (reference src/optimize_op_gpu.cu:891-982  blocksparse_norm)
//   l2_decay_kernel          w -= w * min(rate / sqrt(sum w^2 + eps), 1)          (:794-884  blocksparse_l2_decay)
//   threshold_prune_kernel   gate[b] = norm(b) < threshold ? 0 : 1               (:1006-1098 blocksparse_threshold_prune)
//   prune_topk_kernel        gate[idx[i]] = i < keep                             (:985-1003  blocksparse_prune)
//   identity_init_kernel     W[b] = scale * I on the wrapped diagonal            (src/blocksparse_matmul_op_gpu.cu:2988-3028)
//   l2_normalize_kernel      y = gain * w / sqrt(max(sum_col w^2, eps)) over each OUTPUT feature of a block column
//                            (src/blocksparse_l2_norm_op_gpu.cu:150-234) and its gradient (:593-708)
//   feature_reduce_kernel +  block-reduced full dW for network growth: per-block max|x| / l2 over the feature axis, then a
//   reduced_gemm kernels     dense (bC x bK) product over minibatch x pairs      (src/blocksparse_matmul_op.cc:639-773)
//   gather_rows_kernel ...   SparseProj gather / scatter / scatter_add / scatter_mul (blocksparse/matmul.py:835-921)
#pragma once
#include "common.cuh"

namespace bsmm {

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// One warp per block: lane l walks the block's elements l, l + 32, ... (fully coalesced 64 / 128-byte warp accesses).
template <typename T>
__device__ __forceinline__ void block_reduce(const T* __restrict__ w, int n, int lane, float& max_abs, float& sum_sq) {
  float m = 0.f, s = 0.f;
  for (int i = lane; i < n; i += 32) {
    const float v = to_f32(w[i]);
    m = fmaxf(m, fabsf(v));
    s += v * v;
  }
  max_abs = warp_max(m);
  sum_sq = warp_sum(s);
}

template <typename T>
__global__ void block_norm_kernel(const T* __restrict__ w, float* __restrict__ norm, int blocks, int n, int l2) {
  const int b = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32, lane = threadIdx.x % 32;
  if (b >= blocks) return;
  float m, s;
  block_reduce(w + (size_t)b * n, n, lane, m, s);
  if (lane == 0) norm[b] = l2 ? sqrtf(s) : m;
}

template <typename T>
__global__ void l2_decay_kernel(T* __restrict__ w, const float* __restrict__ gate, int blocks, int n, float rate, float epsilon) {
  const int b = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32, lane = threadIdx.x % 32;
  if (b >= blocks) return;
  if (gate != nullptr && gate[b] == 0.0f) return;           // pruned blocks are left alone
  T* wb = w + (size_t)b * n;
  float m, s;
  block_reduce(wb, n, lane, m, s);
  const float decay = fminf(rsqrtf(s + epsilon) * rate, 1.0f);
  for (int i = lane; i < n; i += 32) {
    const float v = to_f32(wb[i]);
    wb[i] = from_f32<T>(v - v * decay);
  }
}

template <typename T>
__global__ void threshold_prune_kernel(const T* __restrict__ w, float* __restrict__ gate, int blocks, int n, float threshold, int l2) {
  const int b = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32, lane = threadIdx.x % 32;
  if (b >= blocks) return;
  float m, s;
  block_reduce(w + (size_t)b * n, n, lane, m, s);
  if (lane == 0) gate[b] = (l2 ? sqrtf(s) : m) < threshold ? 0.0f : 1.0f;
}

__global__ void prune_topk_kernel(float* __restrict__ gate, const int* __restrict__ idx, int blocks, int keep) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < blocks; i += gridDim.x * blockDim.x) gate[idx[i]] = i < keep ? 1.0f : 0.0f;
}

template <typename T>
__global__ void identity_init_kernel(T* __restrict__ w, const int32_t* __restrict__ updat_lut, int blocks, int bs, int CB, int KB, float scale) {
  const int b = blockIdx.x;
  const int cb = updat_lut[2 * b], kb = updat_lut[2 * b + 1];
  const bool diag = (cb % KB) == (kb % CB);
  T* wb = w + (size_t)b * bs * bs;
  for (int i = threadIdx.x; i < bs * bs; i += blockDim.x)
    wb[i] = from_f32<T>((diag && i / bs == i % bs) ? scale : 0.0f);
}

// ---- l2 normalisation over the columns of the sparse matrix -------------------------------------------------------
// One CTA of 128 threads per output block column k.  Thread (r, j) = (tid / bs, tid % bs) owns output feature j and the
// rows r, r + R, ... (R = 128 / bs row groups) of every block of the column, so a warp reads whole contiguous rows.
// `lut` is the row LUT of fprop (header (first_row, n) per output block, entries (w_block, in_block)).
constexpr int L2N_THREADS = 128;

template <typename T, typename TY>
__global__ void __launch_bounds__(L2N_THREADS)
l2_normalize_kernel(const T* __restrict__ w, const float* __restrict__ gain, TY* __restrict__ y, float* __restrict__ sum_sqr,
                    const int32_t* __restrict__ lut, int bs, float epsilon) {
  __shared__ float red[L2N_THREADS];
  const int k = blockIdx.x, tid = threadIdx.x;
  const int R = L2N_THREADS / bs, j = tid % bs, r0 = tid / bs;
  const int first = lut[2 * k], n = lut[2 * k + 1];
  const int32_t* ent = lut + 2 * first;
  float s = 0.f;
  for (int e = 0; e < n; ++e) {
    const T* wb = w + (size_t)ent[2 * e] * bs * bs;
    for (int i = r0; i < bs; i += R) { const float v = to_f32(wb[i * bs + j]); s += v * v; }
  }
  red[tid] = s;
  __syncthreads();
  if (tid < bs) {
    float t = 0.f;
    for (int r = 0; r < R; ++r) t += red[r * bs + tid];      // fixed order: deterministic
    red[tid] = t;
    sum_sqr[k * bs + tid] = t;
  }
  __syncthreads();
  const float rnorm = rsqrtf(fmaxf(red[j], epsilon)) * (gain ? gain[k * bs + j] : 1.0f);
  for (int e = 0; e < n; ++e) {
    const size_t off = (size_t)ent[2 * e] * bs * bs;
    for (int i = r0; i < bs; i += R) y[off + i * bs + j] = from_f32<TY>(to_f32(w[off + i * bs + j]) * rnorm);
  }
}

// grad_x = (grad_y * g + x * (sum_sqr >= eps) * sum(-grad_y * g * x / norm^2)) / norm ;  grad_g = sum(grad_y * x / norm)
template <typename T, typename TY>
__global__ void __launch_bounds__(L2N_THREADS)
l2_normalize_grad_kernel(const TY* __restrict__ dy, const T* __restrict__ w, const float* __restrict__ gain, const float* __restrict__ sum_sqr,
                         T* __restrict__ dx, float* __restrict__ dg, const int32_t* __restrict__ lut, int bs, float epsilon) {
  __shared__ float red1[L2N_THREADS], red2[L2N_THREADS];
  const int k = blockIdx.x, tid = threadIdx.x;
  const int R = L2N_THREADS / bs, j = tid % bs, r0 = tid / bs;
  const int first = lut[2 * k], n = lut[2 * k + 1];
  const int32_t* ent = lut + 2 * first;
  const float g = gain ? gain[k * bs + j] : 1.0f;
  const float ss = sum_sqr[k * bs + j];
  const float mx = fmaxf(ss, epsilon);
  const float norm_i = rsqrtf(mx), norm2_i = 1.0f / mx;
  float rv = 0.f, dgv = 0.f;
  for (int e = 0; e < n; ++e) {
    const size_t off = (size_t)ent[2 * e] * bs * bs;
    for (int i = r0; i < bs; i += R) {
      const float x = to_f32(w[off + i * bs + j]), d = to_f32(dy[off + i * bs + j]);
      rv += (-d * g * x) * norm2_i;
      dgv += d * x * norm_i;
    }
  }
  red1[tid] = rv; red2[tid] = dgv;
  __syncthreads();
  if (tid < bs) {
    float a = 0.f, b = 0.f;
    for (int r = 0; r < R; ++r) { a += red1[r * bs + tid]; b += red2[r * bs + tid]; }
    red1[tid] = a;
    if (dg) dg[k * bs + tid] = b;
  }
  __syncthreads();
  const float red_val = red1[j] * (ss >= epsilon ? 1.0f : 0.0f);
  for (int e = 0; e < n; ++e) {
    const size_t off = (size_t)ent[2 * e] * bs * bs;
    for (int i = r0; i < bs; i += R) {
      const float x = to_f32(w[off + i * bs + j]), d = to_f32(dy[off + i * bs + j]);
      dx[off + i * bs + j] = from_f32<T>((d * g + x * red_val) * norm_i);
    }
  }
}

// ---- block-reduced full dW ------------------------------------------------------------------------------------------
// x_red: axis 1 -> (pair, n, block) ; axis 0 -> (block, pair, n).  norm_type 0 = max|x|, 1 = l2 over the bs features of a block.
template <typename T>
__global__ void feature_reduce_kernel(const T* __restrict__ x, T* __restrict__ out, int axis, int bs, int nb, int N, int pair, int pcount, int l2) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)nb * N) return;
  float m = 0.f, s = 0.f;
  if (axis == 1) {                 // x (N, nb*bs): thread = (n, block), bs contiguous elements
    const int b = idx % nb; const long long n = idx / nb;
    const T* p = x + n * (long long)nb * bs + (long long)b * bs;
    for (int i = 0; i < bs; ++i) { const float v = to_f32(p[i]); m = fmaxf(m, fabsf(v)); s += v * v; }
    out[((long long)pair * N + n) * nb + b] = from_f32<T>(l2 ? sqrtf(s) : m);
  } else {                         // x (nb*bs, N): thread = (block, n), consecutive threads = consecutive n (coalesced rows)
    const long long n = idx % N; const int b = idx / N;
    const T* p = x + (long long)b * bs * N + n;
    for (int i = 0; i < bs; ++i) { const float v = to_f32(p[(long long)i * N]); m = fmaxf(m, fabsf(v)); s += v * v; }
    out[((long long)b * pcount + pair) * N + n] = from_f32<T>(l2 ? sqrtf(s) : m);
  }
}

// partial[split][i][j] = sum over this split's rows r of A(r, i) * B(r, j); A(r,i) = a[r*a_sr + i*a_si] (same for B).
// 16 x 16 output tile per CTA (256 threads), rows staged 64 at a time through shared memory.
template <typename T>
__global__ void __launch_bounds__(256)
reduced_gemm_partial_kernel(const T* __restrict__ a, const T* __restrict__ b, float* __restrict__ partial, int M, int Nn, long long R,
                            long long a_sr, long long a_si, long long b_sr, long long b_sj, int splits) {
  __shared__ float sa[64][17], sb[64][17];
  const int ti = threadIdx.x / 16, tj = threadIdx.x % 16;
  const int i0 = blockIdx.x * 16, j0 = blockIdx.y * 16, sp = blockIdx.z;
  const long long r_begin = R * sp / splits, r_end = R * (sp + 1) / splits;
  float acc = 0.f;
  for (long long r = r_begin; r < r_end; r += 64) {
    for (int q = threadIdx.x; q < 64 * 16; q += 256) {
      const int rr = q / 16, c = q % 16;
      const long long row = r + rr;
      sa[rr][c] = (row < r_end && i0 + c < M) ? to_f32(a[row * a_sr + (long long)(i0 + c) * a_si]) : 0.f;
      sb[rr][c] = (row < r_end && j0 + c < Nn) ? to_f32(b[row * b_sr + (long long)(j0 + c) * b_sj]) : 0.f;
    }
    __syncthreads();
#pragma unroll 16
    for (int rr = 0; rr < 64; ++rr) acc += sa[rr][ti] * sb[rr][tj];
    __syncthreads();
  }
  if (i0 + ti < M && j0 + tj < Nn) partial[((long long)sp * M + i0 + ti) * Nn + j0 + tj] = acc;
}
__global__ void reduced_gemm_finish_kernel(const float* __restrict__ partial, float* __restrict__ dw, int total, int splits, float scale, int accumulate) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  float s = 0.f;
  for (int sp = 0; sp < splits; ++sp) s += partial[(long long)sp * total + i];       // fixed order
  dw[i] = s * scale + (accumulate ? dw[i] : 0.f);
}

// ---- SparseProj: row gather / scatter on (features, N) activations --------------------------------------------------
// op 0: out[r,:] = idx[r] >= 0 ? x[idx[r],:] : 0            (gather with gather_lut, scatter with scatter_lut)
// op 1: out[r,:] = x[r,:] + (idx[r] >= 0 ? y[idx[r],:] : 0)  (scatter_add; idx = scatter_lut)
// op 2: out[r,:] = x[r,:] * (idx[r] >= 0 ? y[idx[r],:] : 1)  (scatter_mul)
// The row comes from blockIdx.x (up to 2^31 - 1 rows; gridDim.y stops at 65535) and blockIdx.y grid-strides over N.
template <typename T>
__global__ void gather_rows_kernel(const T* __restrict__ x, const T* __restrict__ y, const int32_t* __restrict__ idx, T* __restrict__ out,
                                   int rows, long long N, int op) {
  const int r = blockIdx.x;
  if (r >= rows) return;
  const int src = idx[r];
  for (long long n = (long long)blockIdx.y * blockDim.x + threadIdx.x; n < N; n += (long long)gridDim.y * blockDim.x) {
    float v;
    if (op == 0) v = src >= 0 ? to_f32(x[(long long)src * N + n]) : 0.f;
    else {
      const float a = to_f32(x[(long long)r * N + n]);
      const float b = src >= 0 ? to_f32(y[(long long)src * N + n]) : (op == 1 ? 0.f : 1.f);
      v = op == 1 ? a + b : a * b;
    }
    out[(long long)r * N + n] = from_f32<T>(v);
  }
}

// ---- 8 x 8 blocks on the tensor cores: pad 2 x 2 neighbourhoods into 16 x 16 blocks ---------------------------------
// wgmma needs K = 16 per step, so an 8 x 8 block cannot be an operand on its own.  The host layer builds a SHADOW layout of
// 16 x 16 super-blocks (one per 2 x 2 neighbourhood that holds at least one 8 x 8 block), these kernels scatter the weights
// into it (absent sub-blocks are zero, the optional gate is folded in) and gather the weight gradient back out.  The padded
// product multiplies zeros -- at 20 % density about a third of the super-block is real -- but runs on the tensor cores
// instead of the CUDA-core FMA kernels.
template <typename T>
__global__ void pad_blocks_kernel(const T* __restrict__ w_small, const int32_t* __restrict__ sub_map, const float* __restrict__ gate,
                                  T* __restrict__ w_big, int blocks_big, int bs) {
  const int B = 2 * bs, n = B * B;
  const int b = blockIdx.x;
  for (int idx = threadIdx.x; idx < n; idx += blockDim.x) {
    const int i = idx / B, j = idx % B;
    const int src = sub_map[4 * b + (i / bs) * 2 + (j / bs)];
    float v = 0.f;
    if (src >= 0) {
      v = to_f32(w_small[((size_t)src * bs + (i % bs)) * bs + (j % bs)]);
      if (gate) v *= gate[src];
    }
    w_big[(size_t)b * n + idx] = from_f32<T>(v);
  }
}
// inv_map[w] = super-block id * 4 + sub-position
template <typename TI, typename TO>
__global__ void unpad_blocks_kernel(const TI* __restrict__ dw_big, const int32_t* __restrict__ inv_map, const float* __restrict__ gate,
                                    TO* __restrict__ dw_small, int blocks_small, int bs, int accumulate) {
  const int B = 2 * bs;
  const int w = blockIdx.x;
  const int m = inv_map[w], big = m >> 2, sub = m & 3;
  const TI* src = dw_big + (size_t)big * B * B + (size_t)(sub >> 1) * bs * B + (sub & 1) * bs;
  for (int idx = threadIdx.x; idx < bs * bs; idx += blockDim.x) {
    const int i = idx / bs, j = idx % bs;
    float v = to_f32(src[i * B + j]);
    if (gate) v *= gate[w];                        // gated dW (reference op.cc:274), applied before the output rounding
    if (accumulate) v += to_f32(dw_small[(size_t)w * bs * bs + idx]);
    dw_small[(size_t)w * bs * bs + idx] = from_f32<TO>(v);
  }
}

}  // namespace bsmm
