// Block-sparse convolution (the reference's BlocksparseConv / BlocksparseDeconv) as implicit GEMMs, one per block, on
// sm_90a: bsmm_conv_xprop (fprop / bprop), bsmm_conv_updat and bsmm_conv_l2_normalize(_grad).
//
// Every op is a GEMM whose operands are gathered on the fly through host-built tables:
//   xprop   Y[n, out_ch[c], p] (+)= sum_{j, t} X[n, red_ch[j], lut[p, t]] * F[f_off + c * so + j * sr + t]
//           rows m = (n, p) over N * P_out, columns c over the block's out_len, reduction k = (j, t) over red_len * trs;
//   updat   dF[f_off + o * so + j * sr + t] = sum_{n, p} E[n, out_ch[o], p] * X[n, red_ch[j], lut[p, t]]
//           rows o over out_len, columns (j, t), reduction over the rows (n, p) of one fixed-size chunk.
// lut[p, t] is the input position that output position p reads through tap t, or -1 (padding, or a stride hole in
// bprop). fprop uses the conv's K list as out and C as red (so = C_b trs, sr = trs); bprop swaps them (so = trs,
// sr = C_b trs) with its own lut, so the filter is never flipped or copied. The deconv is the same three ops with the
// roles swapped on the host.
//
// Two kernel families share the operand gathers (XpropOp, UpdatOp):
//   conv_tc_kernel   one warpgroup, 64 x 64 output tile, K steps of 32 staged to shared memory in the no-swizzle
//                    core-matrix layout and multiplied by two wgmma m64n64k16 (fp16 / bf16, fp32 accumulators); the
//                    gathers of step i + 1 are issued into registers while the MMAs of step i run;
//   conv_fma_kernel  256 threads, 64 x 64 tile, 4 x 4 fp32 FMA per thread, any dtype mix (true fp32, no TF32).
// Determinism: every output element is summed by one thread in a fixed k order. Blocks that share output channels run
// in fixed-order passes (host-built; within a pass no two blocks share a channel) that add into one fp32 buffer, rounded
// once at the end. updat writes per-chunk fp32 partials that conv_updat_reduce adds in chunk order. Grids depend on the
// shapes only, never on the SM count.
#pragma once
#include <type_traits>
#include "common.cuh"
#include "ptx.cuh"

namespace bsmm {

// Block record, int32 x 8: out_len, red_len, out channel list offset, red channel list offset, filter offset, so, sr, 0.
struct ConvBlk { int out_len, red_len, out_ch, red_ch, f_off, so, sr, pad; };

constexpr int CONV_T = 64;            // output tile edge (rows and columns)
constexpr int CONV_CHUNK = 8192;      // updat rows per partial sum: fixed, so the sum order never depends on the GPU

struct ConvArgs {
  const ConvBlk* blk;      // this launch's blocks
  const int32_t* ch;       // channel lists
  const int32_t* lut;      // [P_out][trs]
  const void* x;           // gathered activations [N][C_in][P_in]
  const void* f;           // xprop: filter; updat: E [N][C_out][P_out]
  void* y;                 // xprop: output [N][C_out][P_out] (T of x) or fp32 accumulator; updat: fp32 partials
  long long N, P_in, P_out, rows;   // rows: N * P_out
  int C_in, C_out, trs, col_tiles, row_tiles, accumulate;
  long long size_f;
};

// ---- xprop operands: A[m][k] = X gathered, B[n][k] = F ---------------------------------------------------------------
template <typename TX, typename TF, int BK>
struct XpropOp {
  static constexpr bool FAST_K = false;
  struct Smem { long long xrow[CONV_T], yrow[CONV_T], kx[BK]; int lrow[CONV_T], fcol[CONV_T], ycol[CONV_T], kt[BK], kf[BK]; };
  const ConvArgs& a;
  ConvBlk b;
  long long m0;
  int n0, K;
  Smem& s;
  __device__ XpropOp(const ConvArgs& args, Smem& sm, bool& skip) : a(args), s(sm) {
    const int bi = blockIdx.y / args.col_tiles;
    b = args.blk[bi];
    n0 = (blockIdx.y % args.col_tiles) * CONV_T;
    m0 = (long long)blockIdx.x * CONV_T;
    K = b.red_len * args.trs;
    skip = n0 >= b.out_len;
  }
  __device__ void prep_mn() {
    const int i = threadIdx.x;
    if (i < CONV_T) {
      const long long m = m0 + i;
      if (m < a.rows) {
        const long long n = m / a.P_out, p = m - n * a.P_out;
        s.xrow[i] = n * a.C_in * a.P_in;
        s.yrow[i] = n * a.C_out * a.P_out + p;
        s.lrow[i] = (int)p * a.trs;
      } else {
        s.lrow[i] = -1;
      }
    } else if (i < 2 * CONV_T) {
      const int c = n0 + i - CONV_T;
      const bool ok = c < b.out_len;
      s.fcol[i - CONV_T] = ok ? b.f_off + c * b.so : -1;
      s.ycol[i - CONV_T] = ok ? a.ch[b.out_ch + c] : -1;
    }
  }
  __device__ void prep_k(int k0) {
    const int i = threadIdx.x;
    if (i < BK) {
      const int k = k0 + i;
      if (k < K) {
        const int j = k / a.trs, t = k - j * a.trs;
        s.kx[i] = (long long)a.ch[b.red_ch + j] * a.P_in;
        s.kt[i] = t;
        s.kf[i] = j * b.sr + t;
      } else {
        s.kt[i] = -1;
      }
    }
  }
  __device__ float load_a(int m, int k) const {
    const int lr = s.lrow[m], t = s.kt[k];
    if (lr < 0 || t < 0) return 0.f;
    const int g = __ldg(a.lut + lr + t);
    return g < 0 ? 0.f : to_f32(__ldg(static_cast<const TX*>(a.x) + s.xrow[m] + s.kx[k] + g));
  }
  __device__ float load_b(int n, int k) const {
    const int fc = s.fcol[n], t = s.kt[k];
    if (fc < 0 || t < 0) return 0.f;
    return to_f32(__ldg(static_cast<const TF*>(a.f) + fc + s.kf[k]));
  }
  __device__ void store(int m, int n, float v) const {
    if (s.lrow[m] < 0 || s.ycol[n] < 0) return;
    const long long o = s.yrow[m] + (long long)s.ycol[n] * a.P_out;
    if (a.accumulate) static_cast<float*>(a.y)[o] += v;
    else static_cast<TX*>(a.y)[o] = from_f32<TX>(v);
  }
};

// ---- updat operands: A[o][r] = E, B[(j, t)][r] = X gathered; the reduction runs over the chunk's rows r = (n, p) ----
template <typename TE, typename TX, int BK>
struct UpdatOp {
  static constexpr bool FAST_K = true;
  struct Smem { long long ecol[CONV_T], xcol[CONV_T], ke[BK], kx[BK]; int tcol[CONV_T], kl[BK]; };
  const ConvArgs& a;
  ConvBlk b;
  int m0, n0, K, N_;
  long long r0;
  Smem& s;
  __device__ UpdatOp(const ConvArgs& args, Smem& sm, bool& skip) : a(args), s(sm) {
    const int tiles = args.row_tiles * args.col_tiles;
    const int bi = blockIdx.x / tiles, tile = blockIdx.x % tiles;
    b = args.blk[bi];
    m0 = (tile / args.col_tiles) * CONV_T;
    n0 = (tile % args.col_tiles) * CONV_T;
    N_ = b.red_len * args.trs;
    r0 = (long long)blockIdx.y * CONV_CHUNK;
    const long long left = args.rows - r0;
    K = left < CONV_CHUNK ? (int)left : CONV_CHUNK;
    skip = m0 >= b.out_len || n0 >= N_;
  }
  __device__ void prep_mn() {
    const int i = threadIdx.x;
    if (i < CONV_T) {
      const int o = m0 + i;
      s.ecol[i] = o < b.out_len ? (long long)a.ch[b.out_ch + o] * a.P_out : -1;
    } else if (i < 2 * CONV_T) {
      const int jt = n0 + i - CONV_T;
      if (jt < N_) {
        const int j = jt / a.trs;
        s.xcol[i - CONV_T] = (long long)a.ch[b.red_ch + j] * a.P_in;
        s.tcol[i - CONV_T] = jt - j * a.trs;
      } else {
        s.tcol[i - CONV_T] = -1;
      }
    }
  }
  __device__ void prep_k(int k0) {
    const int i = threadIdx.x;
    if (i < BK) {
      const int k = k0 + i;
      if (k < K) {
        const long long r = r0 + k, n = r / a.P_out, p = r - n * a.P_out;
        s.ke[i] = n * a.C_out * a.P_out + p;
        s.kx[i] = n * a.C_in * a.P_in;
        s.kl[i] = (int)p * a.trs;
      } else {
        s.kl[i] = -1;
      }
    }
  }
  __device__ float load_a(int m, int k) const {
    if (s.ecol[m] < 0 || s.kl[k] < 0) return 0.f;
    return to_f32(__ldg(static_cast<const TE*>(a.f) + s.ke[k] + s.ecol[m]));
  }
  __device__ float load_b(int n, int k) const {
    const int t = s.tcol[n], lr = s.kl[k];
    if (t < 0 || lr < 0) return 0.f;
    const int g = __ldg(a.lut + lr + t);
    return g < 0 ? 0.f : to_f32(__ldg(static_cast<const TX*>(a.x) + s.kx[k] + s.xcol[n] + g));
  }
  __device__ void store(int m, int n, float v) const {
    const int o = m0 + m, jt = n0 + n;
    if (o >= b.out_len || jt >= N_) return;
    static_cast<float*>(a.y)[blockIdx.y * a.size_f + b.f_off + (long long)o * b.so + jt] = v;
  }
};

// Tile element e (of 64 x BK) of thread slot i: FAST_K ops walk k fastest (their gathers are contiguous along the rows
// of the reduction), the others m fastest.
template <class Op, int NT, int BK>
__device__ __forceinline__ void conv_mk(int i, int& m, int& k) {
  const int e = threadIdx.x + NT * i;
  if constexpr (Op::FAST_K) { k = e % BK; m = e / BK; }
  else { m = e % CONV_T; k = e / CONV_T; }
}

// ---- CUDA-core kernel -----------------------------------------------------------------------------------------------
template <class Op>
__global__ void __launch_bounds__(256) conv_fma_kernel(const ConvArgs args) {
  constexpr int NT = 256, BK = 16, E = CONV_T * BK / NT;
  __shared__ typename Op::Smem sm;
  __shared__ float As[BK][CONV_T], Bs[BK][CONV_T];
  bool skip;
  Op op(args, sm, skip);
  if (skip) return;
  op.prep_mn();
  const int tx = threadIdx.x % 16, ty = threadIdx.x / 16;
  float acc[4][4] = {};
  for (int k0 = 0; k0 < op.K; k0 += BK) {
    op.prep_k(k0);
    __syncthreads();
#pragma unroll
    for (int i = 0; i < E; ++i) {
      int m, k;
      conv_mk<Op, NT, BK>(i, m, k);
      As[k][m] = op.load_a(m, k);
      Bs[k][m] = op.load_b(m, k);
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < BK; ++k) {
      float av[4], bv[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) { av[i] = As[k][ty + 16 * i]; bv[i] = Bs[k][tx + 16 * i]; }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) op.store(ty + 16 * i, tx + 16 * j, acc[i][j]);
}

// ---- wgmma kernel -----------------------------------------------------------------------------------------------------
// Shared tiles are 64 rows x BK k of T in the canonical no-swizzle K-major layout: core matrices of 8 rows x 8 k
// (128 bytes), the BK / 8 of one 8-row group adjacent along k (leading byte offset 128), 8-row groups BK * 16 bytes
// apart (stride byte offset). A K = 16 step starts 256 bytes further on. BK = 32 keeps the gathers of the next step
// (2 x 16 values per thread) in registers without spilling.
constexpr int CONV_TC_BK = 32;
__device__ __forceinline__ int conv_tc_off(int m, int k) {
  return ((m >> 3) * (CONV_TC_BK / 8) + (k >> 3)) * 64 + (m & 7) * 8 + (k & 7);
}

template <bool BF16, class Op>
__global__ void __launch_bounds__(128) conv_tc_kernel(const ConvArgs args) {
  using T = typename std::conditional<BF16, __nv_bfloat16, __half>::type;
  constexpr int NT = 128, BK = CONV_TC_BK, E = CONV_T * BK / NT;
  __shared__ typename Op::Smem sm;
  __shared__ __align__(128) T As[CONV_T * BK];
  __shared__ __align__(128) T Bs[CONV_T * BK];
  bool skip;
  Op op(args, sm, skip);
  if (skip) return;
  op.prep_mn();
  float d[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) d[i] = 0.f;
  T ra[E], rb[E];
  auto fetch = [&]() {
#pragma unroll
    for (int i = 0; i < E; ++i) {
      int m, k;
      conv_mk<Op, NT, BK>(i, m, k);
      ra[i] = from_f32<T>(op.load_a(m, k));
      rb[i] = from_f32<T>(op.load_b(m, k));
    }
  };
  op.prep_k(0);
  __syncthreads();
  fetch();
  const uint32_t a0 = ptx::smem_u32(As), b0 = ptx::smem_u32(Bs);
  for (int k0 = 0; k0 < op.K; k0 += BK) {
#pragma unroll
    for (int i = 0; i < E; ++i) {
      int m, k;
      conv_mk<Op, NT, BK>(i, m, k);
      As[conv_tc_off(m, k)] = ra[i];
      Bs[conv_tc_off(m, k)] = rb[i];
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy stores -> visible to wgmma
    __syncthreads();
    ptx::wg_fence();
    ptx::wg_fence_regs(d);
#pragma unroll
    for (int s = 0; s < BK / 16; ++s)
      ptx::wgmma<BF16, 0, 0, 64>(d, ptx::make_desc(a0 + 256 * s, 128, BK * 16, ptx::SWZ_NONE),
                                 ptx::make_desc(b0 + 256 * s, 128, BK * 16, ptx::SWZ_NONE));
    ptx::wg_commit();
    if (k0 + BK < op.K) {             // the next step's gathers overlap the MMAs
      op.prep_k(k0 + BK);             // (the k tables are read only by fetch, which finished before the barrier)
      __syncthreads();
      fetch();
    }
    ptx::wg_wait<0>();
    ptx::wg_fence_regs(d);
    __syncthreads();
  }
  // d[4j + 2h + e] = D[16w + l/4 + 8h][8j + 2(l%4) + e]
  const int w = threadIdx.x / 32, l = threadIdx.x % 32;
#pragma unroll
  for (int j = 0; j < 8; ++j)
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int e = 0; e < 2; ++e) op.store(16 * w + l / 4 + 8 * h, 8 * j + 2 * (l % 4) + e, d[4 * j + 2 * h + e]);
}

// dF[e] = sum over chunks c, in order, of partial[c][e], rounded once to TF.
template <typename TF>
__global__ void __launch_bounds__(256) conv_updat_reduce(const float* __restrict__ part, TF* __restrict__ df,
                                                         long long size_f, int chunks) {
  for (long long e = (long long)blockIdx.x * 256 + threadIdx.x; e < size_f; e += (long long)gridDim.x * 256) {
    float s = 0.f;
    for (int c = 0; c < chunks; ++c) s += part[c * size_f + e];
    df[e] = from_f32<TF>(s);
  }
}

// ---- l2 normalisation of filter rows ---------------------------------------------------------------------------------
// Row r (int32 x 4: base, outer, stride, 0) holds x[base + i * stride + t] for i < outer, t < trs: one output channel
// of a block for KCTRS (stride = trs), one input channel for CKTRS (stride = C_b trs). One warp per row; each lane sums
// a fixed set of elements and the lanes are combined by a fixed butterfly, so the result is bitwise reproducible.
struct ConvNormRow { int base, outer, stride, pad; };
constexpr int CN_WARPS = 4;

__device__ __forceinline__ long long cn_off(const ConvNormRow& r, int e, int trs) {
  const int i = e / trs;
  return (long long)r.base + (long long)i * r.stride + (e - i * trs);
}

template <typename TX, typename TY>
__global__ void __launch_bounds__(32 * CN_WARPS) conv_l2n_kernel(const ConvNormRow* rows, int n_rows, int trs,
                                                                 const TX* x, const float* gain, TY* y, float* ss,
                                                                 float epsilon) {
  const int row = blockIdx.x * CN_WARPS + threadIdx.x / 32, lane = threadIdx.x % 32;
  if (row >= n_rows) return;
  const ConvNormRow r = rows[row];
  const int len = r.outer * trs;
  float s = 0.f;
  for (int e = lane; e < len; e += 32) {
    const float v = to_f32(x[cn_off(r, e, trs)]);
    s = fmaf(v, v, s);
  }
#pragma unroll
  for (int i = 16; i > 0; i >>= 1) s += __shfl_xor_sync(0xffffffffu, s, i);
  if (lane == 0) ss[row] = s;
  const float rn = (gain ? gain[row] : 1.f) / sqrtf(fmaxf(s, epsilon));
  for (int e = lane; e < len; e += 32) {
    const long long o = cn_off(r, e, trs);
    y[o] = from_f32<TY>(to_f32(x[o]) * rn);
  }
}

// dx = (dy g - x [ss >= eps] g sum(dy x) / max(ss, eps)) / sqrt(max(ss, eps)); dg = sum(dy x) / sqrt(max(ss, eps)).
template <typename TX, typename TD>
__global__ void __launch_bounds__(32 * CN_WARPS) conv_l2n_grad_kernel(const ConvNormRow* rows, int n_rows, int trs,
                                                                      const TD* dy, const TX* x, const float* gain,
                                                                      const float* ss, TX* dx, float* dg, float epsilon) {
  const int row = blockIdx.x * CN_WARPS + threadIdx.x / 32, lane = threadIdx.x % 32;
  if (row >= n_rows) return;
  const ConvNormRow r = rows[row];
  const int len = r.outer * trs;
  float s = 0.f;
  for (int e = lane; e < len; e += 32) {
    const long long o = cn_off(r, e, trs);
    s = fmaf(to_f32(dy[o]), to_f32(x[o]), s);
  }
#pragma unroll
  for (int i = 16; i > 0; i >>= 1) s += __shfl_xor_sync(0xffffffffu, s, i);
  const float sq = ss[row], mx = fmaxf(sq, epsilon), rn = 1.f / sqrtf(mx), g = gain ? gain[row] : 1.f;
  if (dg && lane == 0) dg[row] = s * rn;
  const float c = sq >= epsilon ? -s * g / mx : 0.f;
  for (int e = lane; e < len; e += 32) {
    const long long o = cn_off(r, e, trs);
    dx[o] = from_f32<TX>((to_f32(dy[o]) * g + to_f32(x[o]) * c) * rn);
  }
}

}  // namespace bsmm
