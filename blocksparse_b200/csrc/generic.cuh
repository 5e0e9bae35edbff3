// CUDA-core kernel families (fp32 FMA, any storage dtype, block size 8/16/32/64).
//
// These are the true-fp32 path (BASELINE cfg 1, <=1e-5) and the fallback for the
// (dtype, block size, axis) combinations that have no wgmma kernel.  Two shapes
// cover the whole hot path:
//
//   sdd_xn : sparse . dense -> dense     (bsmm fprop/bprop, bst NN/TN)
//            replaces gemm_blocksparse_*_xprop (src/blocksparse_matmul_op_gpu.cu:8-958)
//            and bst_sgemm_32x64x32_xn (src/bst_sgemm_op_gpu.cu:7-231)
//   dds_nt : dense . dense^T -> sparse   (bsmm updat, bst NT)
//            replaces gemm_blocksparse_*_updat (src/blocksparse_matmul_op_gpu.cu:960-1835)
//            and bst_sgemm_32x32x64_nt (src/bst_sgemm_op_gpu.cu:233-416)
//
// Unlike the reference there are no segments, spin locks or atomics: one CTA owns a
// whole (output block, n-tile) and walks the complete LUT row, so results are
// deterministic.
#pragma once
#include "common.cuh"

namespace bsmm {

// ------------------------------------------------------------------------------------
// sdd_xn
// ------------------------------------------------------------------------------------
struct XnParams {
  const int32_t* lut;       // row LUT of lut-head 0: [n_out + nnz][2]
  long long lut_head_stride;  // ints between lut heads (0 = shared)
  int n_out;
  const void* w;            // sparse operand, (.., blocks, BS, BS)
  long long w_z_stride;     // elements between z slices of w (bst: blocks*BS*BS), 0 for bsmm
  const void* x;            // dense input
  void* y;                  // dense output
  long long x_zb, x_zh;     // element offsets per batch / per head for x
  long long y_zb, y_zh;
  long long x_sf, x_sn;     // element strides: feature row, n column
  long long y_sf, y_sn;
  int N;                    // columns (minibatch, or head_state for bst)
  int heads;                // z = b*heads + h
  const float* gate;        // optional per-block scale, 0 => skip
};

template <typename TW, typename TX, int BS, bool FEAT_CONTIG, bool TRANS_W>
__global__ void __launch_bounds__(BS * 4)
sdd_xn_kernel(const XnParams p) {
  constexpr int TN = 64;
  constexpr int NT = BS * 4;
  __shared__ float Ws[BS][BS + 1];
  __shared__ float Xs[BS][TN + 1];

  const int tid = threadIdx.x;
  const int tx = tid % 16;          // n = n0 + tx + 16*j
  const int ty = tid / 16;          // fo = ty*4 + i
  const int n0 = blockIdx.x * TN;
  const int o = blockIdx.y;
  const int z = blockIdx.z;
  const int zb = z / p.heads, zh = z % p.heads;

  const int32_t* lut = p.lut + (long long)zh * p.lut_head_stride;
  const int first = lut[2 * o], count = lut[2 * o + 1];

  const TW* w = reinterpret_cast<const TW*>(p.w) + (long long)z * p.w_z_stride;
  const TX* x = reinterpret_cast<const TX*>(p.x) + zb * p.x_zb + zh * p.x_zh;
  TX* y = reinterpret_cast<TX*>(p.y) + zb * p.y_zb + zh * p.y_zh;

  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  for (int e = 0; e < count; ++e) {
    const int wb = lut[2 * (first + e)];
    const int ib = lut[2 * (first + e) + 1];
    float g = 1.f;
    if (p.gate != nullptr) {
      g = p.gate[wb];
      if (g == 0.f) continue;       // uniform across the CTA
    }
    __syncthreads();
    // W block -> Ws[fi][fo]
    const TW* wblk = w + (long long)wb * BS * BS;
#pragma unroll
    for (int idx = tid; idx < BS * BS; idx += NT) {
      const int i = idx / BS, j = idx % BS;
      const float v = to_f32<TW>(wblk[idx]) * g;
      if (TRANS_W) Ws[j][i] = v; else Ws[i][j] = v;
    }
    // X tile -> Xs[fi][n]
    if (FEAT_CONTIG) {
#pragma unroll
      for (int idx = tid; idx < BS * TN; idx += NT) {
        const int n = idx / BS, fi = idx % BS;
        float v = 0.f;
        if (n0 + n < p.N) v = to_f32<TX>(x[(long long)(ib * BS + fi) * p.x_sf + (long long)(n0 + n) * p.x_sn]);
        Xs[fi][n] = v;
      }
    } else {
#pragma unroll
      for (int idx = tid; idx < BS * TN; idx += NT) {
        const int fi = idx / TN, n = idx % TN;
        float v = 0.f;
        if (n0 + n < p.N) v = to_f32<TX>(x[(long long)(ib * BS + fi) * p.x_sf + (long long)(n0 + n) * p.x_sn]);
        Xs[fi][n] = v;
      }
    }
    __syncthreads();
#pragma unroll 8
    for (int fi = 0; fi < BS; ++fi) {
      float a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) a[i] = Ws[fi][ty * 4 + i];
#pragma unroll
      for (int j = 0; j < 4; ++j) b[j] = Xs[fi][tx + 16 * j];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
  }
  // epilogue (also zero-fills output blocks whose LUT row is empty)
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int fo = ty * 4 + i;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + tx + 16 * j;
      if (n < p.N) y[(long long)(o * BS + fo) * p.y_sf + (long long)n * p.y_sn] = from_f32<TX>(acc[i][j]);
    }
  }
}

template <typename TW, typename TX, int BS>
int launch_sdd_xn(const XnParams& p, bool feat_contig, bool trans_w, int zdim, cudaStream_t s) {
  dim3 grid((p.N + 63) / 64, p.n_out, zdim);
  dim3 block(BS * 4);
  if (feat_contig) {
    if (trans_w) sdd_xn_kernel<TW, TX, BS, true, true><<<grid, block, 0, s>>>(p);
    else         sdd_xn_kernel<TW, TX, BS, true, false><<<grid, block, 0, s>>>(p);
  } else {
    if (trans_w) sdd_xn_kernel<TW, TX, BS, false, true><<<grid, block, 0, s>>>(p);
    else         sdd_xn_kernel<TW, TX, BS, false, false><<<grid, block, 0, s>>>(p);
  }
  return check_launch("fma_sdd_xn");
}

// ------------------------------------------------------------------------------------
// dds_nt
// ------------------------------------------------------------------------------------
struct NtParams {
  const int32_t* lut;         // [blocks][2] = (a_block, b_block), lut-head 0
  long long lut_head_stride;
  int blocks;
  const void* a[BSMM_MAX_PAIRS];
  const void* b[BSMM_MAX_PAIRS];
  int pcount;
  void* out;                  // (.., blocks, BS, BS)
  long long a_zb, a_zh, b_zb, b_zh;   // per batch / per head element offsets
  long long a_sf, a_sr, b_sf, b_sr;   // feature-row stride, reduction stride
  long long out_z_stride;     // elements between z slices of out
  int R;                      // reduction length (minibatch, or head_state)
  int heads;
  float alpha, beta;
  const float* gate;          // only applied when gated
  int gated;
};

template <typename TI, typename TO, int BS, bool FEAT_CONTIG>
__global__ void __launch_bounds__((BS / (BS == 64 ? 4 : 2)) * (BS / (BS == 64 ? 4 : 2)) < 32 ? 32
                                  : (BS / (BS == 64 ? 4 : 2)) * (BS / (BS == 64 ? 4 : 2)))
dds_nt_kernel(const NtParams p) {
  constexpr int PT = (BS == 64) ? 4 : 2;
  constexpr int TD = BS / PT;                  // threads per dim
  constexpr int NT = TD * TD < 32 ? 32 : TD * TD;
  constexpr int RC = 32;
  __shared__ float As[BS][RC + 1];
  __shared__ float Bs[BS][RC + 1];

  const int tid = threadIdx.x;
  const bool active = tid < TD * TD;
  const int tx = tid % TD, ty = (tid / TD) % TD;
  const int blk = blockIdx.x;
  const int z = blockIdx.y;
  const int zb = z / p.heads, zh = z % p.heads;
  const int32_t* lut = p.lut + (long long)zh * p.lut_head_stride;
  const int ab = lut[2 * blk], bb = lut[2 * blk + 1];

  TO* out = reinterpret_cast<TO*>(p.out) + (long long)z * p.out_z_stride + (long long)blk * BS * BS;

  float g = 1.f;
  if (p.gated && p.gate != nullptr) g = p.gate[blk];

  float acc[PT][PT];
#pragma unroll
  for (int u = 0; u < PT; ++u)
#pragma unroll
    for (int v = 0; v < PT; ++v) acc[u][v] = 0.f;

  if (g != 0.f) {
    for (int pi = 0; pi < p.pcount; ++pi) {
      const TI* a = reinterpret_cast<const TI*>(p.a[pi]) + zb * p.a_zb + zh * p.a_zh;
      const TI* b = reinterpret_cast<const TI*>(p.b[pi]) + zb * p.b_zb + zh * p.b_zh;
      for (int r0 = 0; r0 < p.R; r0 += RC) {
        __syncthreads();
        if (FEAT_CONTIG) {
          for (int idx = tid; idx < BS * RC; idx += NT) {
            const int r = idx / BS, f = idx % BS;
            float va = 0.f, vb = 0.f;
            if (r0 + r < p.R) {
              va = to_f32<TI>(a[(long long)(ab * BS + f) * p.a_sf + (long long)(r0 + r) * p.a_sr]);
              vb = to_f32<TI>(b[(long long)(bb * BS + f) * p.b_sf + (long long)(r0 + r) * p.b_sr]);
            }
            As[f][r] = va; Bs[f][r] = vb;
          }
        } else {
          for (int idx = tid; idx < BS * RC; idx += NT) {
            const int f = idx / RC, r = idx % RC;
            float va = 0.f, vb = 0.f;
            if (r0 + r < p.R) {
              va = to_f32<TI>(a[(long long)(ab * BS + f) * p.a_sf + (long long)(r0 + r) * p.a_sr]);
              vb = to_f32<TI>(b[(long long)(bb * BS + f) * p.b_sf + (long long)(r0 + r) * p.b_sr]);
            }
            As[f][r] = va; Bs[f][r] = vb;
          }
        }
        __syncthreads();
        if (active) {
#pragma unroll 8
          for (int r = 0; r < RC; ++r) {
            float av[PT], bv[PT];
#pragma unroll
            for (int u = 0; u < PT; ++u) av[u] = As[ty * PT + u][r];
#pragma unroll
            for (int v = 0; v < PT; ++v) bv[v] = Bs[tx * PT + v][r];
#pragma unroll
            for (int u = 0; u < PT; ++u)
#pragma unroll
              for (int v = 0; v < PT; ++v) acc[u][v] = fmaf(av[u], bv[v], acc[u][v]);
          }
        }
      }
    }
  }
  if (active) {
#pragma unroll
    for (int u = 0; u < PT; ++u)
#pragma unroll
      for (int v = 0; v < PT; ++v) {
        const int i = ty * PT + u, j = tx * PT + v;
        float r = acc[u][v] * p.alpha * g;
        if (p.beta != 0.f) r += p.beta * to_f32<TO>(out[i * BS + j]);
        out[i * BS + j] = from_f32<TO>(r);
      }
  }
}

template <typename TI, typename TO, int BS>
int launch_dds_nt(const NtParams& p, bool feat_contig, int zdim, cudaStream_t s) {
  constexpr int PT = (BS == 64) ? 4 : 2;
  constexpr int TD = BS / PT;
  constexpr int NT = TD * TD < 32 ? 32 : TD * TD;
  dim3 grid(p.blocks, zdim);
  if (feat_contig) dds_nt_kernel<TI, TO, BS, true><<<grid, NT, 0, s>>>(p);
  else             dds_nt_kernel<TI, TO, BS, false><<<grid, NT, 0, s>>>(p);
  return check_launch("fma_dds_nt");
}

// ------------------------------------------------------------------------------------
// gate grad: dg[w] = sum_ij dw[w][i][j] * w[w][i][j]
// ------------------------------------------------------------------------------------
template <typename T>
__global__ void gate_grad_kernel(const T* __restrict__ dw, const T* __restrict__ w, float* __restrict__ dg,
                                 int blocks, int elems) {
  const int blk = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32;
  if (blk >= blocks) return;
  const int lane = threadIdx.x % 32;
  const T* a = dw + (long long)blk * elems;
  const T* b = w + (long long)blk * elems;
  float s = 0.f;
  for (int i = lane; i < elems; i += 32) s = fmaf(to_f32<T>(a[i]), to_f32<T>(b[i]), s);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) dg[blk] = s;
}

// w_out[w] = gate[w] * w[w]  (a zero gate gives an exact zero block).  Lets a gated fprop / bprop of 16-bit weights run
// on the wgmma kernel: the reference's gated tensor-core kernels also scale the loaded 16-bit weights by the gate.
template <typename T>
__global__ void gate_weights_kernel(const T* __restrict__ w, const float* __restrict__ gate, T* __restrict__ out,
                                    long long total, int elems) {
  const long long i = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * 2;
  if (i >= total) return;
  const float g = gate[i / elems];
  out[i] = from_f32<T>(to_f32<T>(w[i]) * g);            // elems is even: both elements belong to the same block
  out[i + 1] = from_f32<T>(to_f32<T>(w[i + 1]) * g);
}

}  // namespace bsmm
