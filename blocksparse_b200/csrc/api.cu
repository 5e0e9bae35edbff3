// C ABI of libbsmm_b200.so -- argument validation and kernel-family dispatch.
// See include/bsmm_b200.h for the contract and the reference launchers each entry replaces.
#include <atomic>
#include <climits>
#include "common.cuh"
#include "conv.cuh"
#include "conv_bias.cuh"
#include "dense_dw.cuh"
#include "dense_softmax.cuh"
#include "elementwise.cuh"
#include "embed.cuh"
#include "ewops.cuh"
#include "generic.cuh"
#include "layer_norm.cuh"
#include "lstm.cuh"
#include "optimize.cuh"
#include "quantize.cuh"
#include "softmax.cuh"
#include "tc.cuh"
#include "tc_bst_decode.cuh"
#include "tc_fp8.cuh"
#include "tc_updat_fp8.cuh"
#include "transpose.cuh"
#include "wutil.cuh"

using namespace bsmm;

extern "C" {

int bsmm_version(void) { return 1000 * 0 + 1; }
const char* bsmm_last_error(void) { return err_buf(); }
const char* bsmm_last_kernel(void) { return kernel_name_slot(); }

int bsmm_device_info(int* sm_count, int* cc_major, int* cc_minor) {
  const DeviceInfo& d = device_info();
  if (!d.ok) return fail(BSMM_E_NODEV, "no CUDA device");
  if (sm_count) *sm_count = d.sm_count;
  if (cc_major) *cc_major = d.cc_major;
  if (cc_minor) *cc_minor = d.cc_minor;
  return 0;
}

int bsmm_device_error(void) {
  int v = 0, zero = 0;
  cudaError_t e = cudaDeviceSynchronize();
  if (e != cudaSuccess) { cudaGetLastError(); fail((int)e, "device fault: %s", cudaGetErrorString(e)); return -1; }
  if (cudaMemcpyFromSymbol(&v, g_tc_error, sizeof(int)) != cudaSuccess) return -1;
  if (v != 0) cudaMemcpyToSymbol(g_tc_error, &zero, sizeof(int));
  int wv = 0;
  if (cudaMemcpyFromSymbol(&wv, ptx::g_wait_error, sizeof(int)) != cudaSuccess) return -1;
  if (wv != 0) cudaMemcpyToSymbol(ptx::g_wait_error, &zero, sizeof(int));
  return v ? v : wv;
}

int bsmm_debug_trace(unsigned long long* out, int n) {
  (void)out; (void)n;
  return fail(BSMM_E_ARG, "bsmm_debug_trace: no kernel of this build records a trace");
}

int bsmm_set_wait_timeout_ms(int ms, int trap) {
  if (ms <= 0) return fail(BSMM_E_ARG, "bsmm_set_wait_timeout_ms: ms must be positive");
  const unsigned long long ns = (unsigned long long)ms * 1000000ull;
  const int t = trap ? 1 : 0;
  cudaError_t e = cudaMemcpyToSymbol(ptx::g_wait_timeout_ns, &ns, sizeof(ns));
  if (e == cudaSuccess) e = cudaMemcpyToSymbol(ptx::g_wait_trap, &t, sizeof(t));
  if (e != cudaSuccess) { cudaGetLastError(); return fail((int)e, "bsmm_set_wait_timeout_ms: %s", cudaGetErrorString(e)); }
  return 0;
}

// ---------------------------------------------------------------------------------------
// A 16-bit call that cannot take the wgmma kernel runs many times slower on the CUDA-core path: say so once per process (the
// reason is whatever tc_* recorded), unless BSMM_QUIET is set.  fp32 calls are expected there and stay silent.
static void note_fallback(const char* op, int dtype) {
  static std::atomic<bool> warned{false};
  if (dtype == BSMM_F32 || warned.exchange(true)) return;
  if (getenv("BSMM_QUIET")) return;
  fprintf(stderr, "[bsmm_b200] %s: no tensor-core kernel for this call (%s); using the CUDA-core FMA kernel (much slower). "
                  "This message is printed once.\n", op, err_buf());
}

static int check_bsize_axis(int bsize, int axis) {
  if (axis != 0 && axis != 1) return fail(BSMM_E_BSIZE, "feature axis must be 0 or 1, got %d", axis);
  if (bsize != 8 && bsize != 16 && bsize != 32 && bsize != 64)
    return fail(BSMM_E_BSIZE, "block size must be 8, 16, 32 or 64, got %d", bsize);
  return 0;
}

int bsmm_xprop(int dtype, int axis, int bsize, int bprop,
               const int32_t* lut, int n_out, int n_in, int blocks,
               const void* x, const void* w, void* y, int N,
               const float* gate,
               const int32_t* sched, int sched_tiles, int sched_tile_blocks, int sched_groups_off,
               int sched_list_off, int sched_ctas, int sched_ntiles,
               int flags, void* stream) {
  if (int e = check_bsize_axis(bsize, axis)) return e;
  if (!lut || !x || !w || !y) return fail(BSMM_E_ARG, "bsmm_xprop: null pointer");
  if (n_out <= 0 || n_in <= 0 || blocks < 0 || N < 0) return fail(BSMM_E_ARG, "bsmm_xprop: bad sizes");
  // reference limit: C, K < bsize*65536 (src/blocksparse_matmul_op.cc:96-97)
  if (n_out >= 65536 || n_in >= 65536) return fail(BSMM_E_LIMIT, "bsmm_xprop: more than 65535 blocks per dimension");
  if (N == 0) return 0;
  cudaStream_t s = (cudaStream_t)stream;

  (void)sched_list_off; (void)sched_ctas; (void)sched_ntiles;
  if (!(flags & BSMM_FLAG_FORCE_GENERIC)) {
    int rc;
    if (((sched_tile_blocks >> 16) & 1) && gate == nullptr)   // wide-tile schedule (lut.py:build_wide_schedule) -> csrc/tc_xprop2.cuh
      rc = tc_xprop2(dtype, axis, bprop, n_out, n_in, blocks, x, w, y, N, sched, sched_tiles, (sched_tile_blocks >> 8) & 0xff,
                     sched_groups_off, s);
    else                                                       // bit 12: 2-CTA clusters sharing the W blocks (pair tiles)
      rc = tc_xprop(dtype, axis, bsize, bprop, lut, n_out, n_in, blocks, x, w, y, N, gate, (sched_tile_blocks >> 12) & 1, s);
    if (rc != TC_NOT_APPLICABLE) return rc;
    if (flags & BSMM_FLAG_FORCE_TC)
      return fail(BSMM_E_ARG, "bsmm_xprop: no wgmma kernel for dtype=%d axis=%d bsize=%d (%s)", dtype, axis, bsize, err_buf());
    note_fallback("bsmm_xprop", dtype);
  } else if (flags & BSMM_FLAG_FORCE_TC) {
    return fail(BSMM_E_ARG, "bsmm_xprop: contradictory flags");
  }

  XnParams p = {};
  p.lut = lut; p.lut_head_stride = 0; p.n_out = n_out;
  p.w = w; p.w_z_stride = 0;
  p.x = x; p.y = y;
  p.heads = 1; p.N = N; p.gate = gate;
  if (axis == 0) { p.x_sf = N; p.x_sn = 1; p.y_sf = N; p.y_sn = 1; }
  else { p.x_sf = 1; p.x_sn = (long long)n_in * bsize; p.y_sf = 1; p.y_sn = (long long)n_out * bsize; }
  // Wm[fi][fo]: fprop uses W[fi][fo] directly, bprop needs the transpose.
  const bool trans_w = bprop != 0;
  BSMM_DISPATCH_DTYPE(dtype, T, {
    BSMM_DISPATCH_BSIZE(bsize, BS, { return launch_sdd_xn<T, T, BS>(p, axis == 1, trans_w, 1, s); });
  });
  return 0;
}

int bsmm_updat(int dtype, int dw_dtype, int axis, int bsize,
               const int32_t* updat_lut, int blocks, int n_c_blocks, int n_k_blocks,
               const void* const* xs, const void* const* dys, int pcount,
               void* dw, int N, float alpha, float beta,
               const float* gate, int gated_dw,
               const int32_t* sched, int sched_tiles, int sched_tile_blocks, int sched_groups_off,
               int flags, void* stream) {
  if (int e = check_bsize_axis(bsize, axis)) return e;
  if (!updat_lut || !xs || !dys || !dw) return fail(BSMM_E_ARG, "bsmm_updat: null pointer");
  if (pcount < 1 || pcount > BSMM_MAX_PAIRS)
    return fail(BSMM_E_ARG, "bsmm_updat: pcount must be in [1,%d], got %d", BSMM_MAX_PAIRS, pcount);
  if (beta != 0.f && beta != 1.f) return fail(BSMM_E_ARG, "bsmm_updat: beta must be 0 or 1");
  if (dw_dtype != dtype && dw_dtype != BSMM_F32) return fail(BSMM_E_DTYPE, "bsmm_updat: dw dtype must be fp32 or the input dtype");
  if (blocks <= 0 || N < 0) return fail(BSMM_E_ARG, "bsmm_updat: bad sizes");
  for (int i = 0; i < pcount; ++i)
    if (!xs[i] || !dys[i]) return fail(BSMM_E_ARG, "bsmm_updat: null pointer in pair %d", i);
  cudaStream_t s = (cudaStream_t)stream;

  if (!(flags & BSMM_FLAG_FORCE_GENERIC)) {
    (void)sched_groups_off;
    int rc = tc_updat(dtype, dw_dtype, axis, bsize, n_c_blocks, n_k_blocks, xs, dys, pcount,
                      dw, N, alpha, beta, gate, gated_dw, sched, sched_tiles, sched_tile_blocks, s);
    if (rc != TC_NOT_APPLICABLE) return rc;
    if (flags & BSMM_FLAG_FORCE_TC)
      return fail(BSMM_E_ARG, "bsmm_updat: no wgmma kernel for dtype=%d axis=%d bsize=%d (%s)", dtype, axis, bsize, err_buf());
    note_fallback("bsmm_updat", dtype);
  }

  NtParams p = {};
  p.lut = updat_lut; p.lut_head_stride = 0; p.blocks = blocks;
  for (int i = 0; i < pcount; ++i) { p.a[i] = xs[i]; p.b[i] = dys[i]; }
  p.pcount = pcount; p.out = dw; p.out_z_stride = 0;
  p.R = N; p.heads = 1; p.alpha = alpha; p.beta = beta; p.gate = gate; p.gated = gated_dw && gate;
  if (axis == 0) { p.a_sf = N; p.a_sr = 1; p.b_sf = N; p.b_sr = 1; }
  else { p.a_sf = 1; p.a_sr = (long long)n_c_blocks * bsize; p.b_sf = 1; p.b_sr = (long long)n_k_blocks * bsize; }
  BSMM_DISPATCH_DTYPE(dtype, T, {
    BSMM_DISPATCH_BSIZE(bsize, BS, {
      if (dw_dtype == BSMM_F32) return launch_dds_nt<T, float, BS>(p, axis == 1, 1, s);
      else                      return launch_dds_nt<T, T, BS>(p, axis == 1, 1, s);
    });
  });
  return 0;
}

int bsmm_gate_grad(int dtype, int bsize, int blocks, const void* dw, const void* w, float* dg, void* stream) {
  if (!dw || !w || !dg || blocks <= 0) return fail(BSMM_E_ARG, "bsmm_gate_grad: bad arguments");
  if (int e = check_bsize_axis(bsize, 0)) return e;
  cudaStream_t s = (cudaStream_t)stream;
  const int warps = 4;
  BSMM_DISPATCH_DTYPE(dtype, T, {
    gate_grad_kernel<T><<<(blocks + warps - 1) / warps, warps * 32, 0, s>>>(
        (const T*)dw, (const T*)w, dg, blocks, bsize * bsize);
  });
  return check_launch("gate_grad");
}

int bsmm_gate_weights(int dtype, int bsize, int blocks, const void* w, const float* gate, void* w_out, void* stream) {
  if (!w || !gate || !w_out || blocks <= 0) return fail(BSMM_E_ARG, "bsmm_gate_weights: bad arguments");
  if (int e = check_bsize_axis(bsize, 0)) return e;
  cudaStream_t s = (cudaStream_t)stream;
  const long long total = (long long)blocks * bsize * bsize;
  const int threads = 256;
  const long long grid = (total / 2 + threads - 1) / threads;
  BSMM_DISPATCH_DTYPE(dtype, T, {
    gate_weights_kernel<T><<<(unsigned)grid, threads, 0, s>>>((const T*)w, gate, (T*)w_out, total, bsize * bsize);
  });
  return check_launch("gate_weights");
}

// ---------------------------------------------------------------------------------------
static int check_bst(int bsize, int lut_heads, int heads, int head_state, int batch, int blocks) {
  if (bsize != 8 && bsize != 16 && bsize != 32 && bsize != 64)
    return fail(BSMM_E_BSIZE, "block size must be 8, 16, 32 or 64, got %d", bsize);
  if (lut_heads != 1 && lut_heads != heads) return fail(BSMM_E_ARG, "lut_heads must be 1 or heads");
  if (batch <= 0 || heads <= 0 || blocks <= 0) return fail(BSMM_E_ARG, "bad batch/heads/blocks");
  if (head_state <= 0 || (head_state & 7)) return fail(BSMM_E_ARG, "head_state must be a positive multiple of 8 (bst_op.cc:208)");
  return 0;
}

int bst_nt(int dtype, int c_dtype, int bsize,
           const int32_t* nt_lut, int lut_heads, int blocks,
           const int32_t* nt_items, int n_items,
           const void* a, const void* b, void* c,
           int batch, int heads, int head_state, int ctx_blks_a, int ctx_blks_b,
           int flags, void* stream) {
  if (int e = check_bst(bsize, lut_heads, heads, head_state, batch, blocks)) return e;
  if (!nt_lut || !a || !b || !c) return fail(BSMM_E_ARG, "bst_nt: null pointer");
  // attention tensor must have < 2^32 elements (bst_op.cc:214)
  if ((unsigned long long)batch * heads * blocks * bsize * bsize >= (1ull << 32))
    return fail(BSMM_E_LIMIT, "bst_nt: output has >= 2^32 elements");
  cudaStream_t s = (cudaStream_t)stream;

  if (!(flags & BSMM_FLAG_FORCE_GENERIC)) {
    (void)nt_items; (void)n_items;
    int rc = tc_bst_nt(dtype, c_dtype, bsize, nt_lut, lut_heads, blocks, a, b, c, batch, heads, head_state,
                       ctx_blks_a, ctx_blks_b, s);
    if (rc != TC_NOT_APPLICABLE) return rc;
    if (flags & BSMM_FLAG_FORCE_TC) return fail(BSMM_E_ARG, "bst_nt: no wgmma kernel for this configuration (%s)", err_buf());
  }

  const long long S = (long long)heads * head_state;
  NtParams p = {};
  p.lut = nt_lut; p.lut_head_stride = lut_heads > 1 ? 2LL * blocks : 0; p.blocks = blocks;
  p.a[0] = a; p.b[0] = b; p.pcount = 1; p.out = c;
  p.a_zb = (long long)ctx_blks_a * bsize * S; p.a_zh = head_state;
  p.b_zb = (long long)ctx_blks_b * bsize * S; p.b_zh = head_state;
  p.a_sf = S; p.a_sr = 1; p.b_sf = S; p.b_sr = 1;
  p.out_z_stride = (long long)blocks * bsize * bsize;
  p.R = head_state; p.heads = heads; p.alpha = 1.f; p.beta = 0.f; p.gate = nullptr; p.gated = 0;
  BSMM_DISPATCH_DTYPE(dtype, T, {
    BSMM_DISPATCH_DTYPE(c_dtype, TC, {
      BSMM_DISPATCH_BSIZE(bsize, BS, { return launch_dds_nt<T, TC, BS>(p, false, batch * heads, s); });
    });
  });
  return 0;
}

int bst_xn(int a_dtype, int dtype, int bsize, int transpose_a,
           const int32_t* lut, const int32_t* out_order, int lut_heads, int blocks, int max_lut,
           const void* a, const void* b, void* c,
           int batch, int heads, int head_state, int ctx_blks_b, int ctx_blks_c,
           int flags, void* stream) {
  if (int e = check_bst(bsize, lut_heads, heads, head_state, batch, blocks)) return e;
  if (!lut || !a || !b || !c) return fail(BSMM_E_ARG, "bst_xn: null pointer");
  cudaStream_t s = (cudaStream_t)stream;

  if (!(flags & BSMM_FLAG_FORCE_GENERIC)) {
    (void)out_order; (void)max_lut;
    int rc = tc_bst_xn(a_dtype, dtype, bsize, transpose_a, lut, lut_heads, blocks, a, b, c, batch, heads,
                       head_state, ctx_blks_b, ctx_blks_c, s);
    if (rc != TC_NOT_APPLICABLE) return rc;
    if (flags & BSMM_FLAG_FORCE_TC) return fail(BSMM_E_ARG, "bst_xn: no wgmma kernel for this configuration (%s)", err_buf());
  }

  const long long S = (long long)heads * head_state;
  XnParams p = {};
  p.lut = lut; p.lut_head_stride = lut_heads > 1 ? 2LL * (ctx_blks_c + blocks) : 0; p.n_out = ctx_blks_c;
  p.w = a; p.w_z_stride = (long long)blocks * bsize * bsize;
  p.x = b; p.y = c;
  p.x_zb = (long long)ctx_blks_b * bsize * S; p.x_zh = head_state;
  p.y_zb = (long long)ctx_blks_c * bsize * S; p.y_zh = head_state;
  p.x_sf = S; p.x_sn = 1; p.y_sf = S; p.y_sn = 1;
  p.N = head_state; p.heads = heads; p.gate = nullptr;
  // NN: out row i of A (fo = i, fi = j) -> transposed staging; TN: fo = j, fi = i -> direct.
  const bool trans_w = transpose_a == 0;
  BSMM_DISPATCH_DTYPE(a_dtype, TA, {
    BSMM_DISPATCH_DTYPE(dtype, T, {
      BSMM_DISPATCH_BSIZE(bsize, BS, { return launch_sdd_xn<TA, T, BS>(p, false, trans_w, batch * heads, s); });
    });
  });
  return 0;
}

int bst_softmax(int x_dtype, int y_dtype, int bsize,
                const int32_t* nn_lut, const int32_t* nt_lut, int lut_heads, int blocks, int max_lut,
                const void* mask, int mask_heads, int autoregress_at_key,
                const void* x, void* y, float scale,
                int batch, int heads, int ctx_blks_q, void* stream) {
  if (int e = check_bst(bsize, lut_heads, heads, 8, batch, blocks)) return e;
  if (!nn_lut || !x || !y) return fail(BSMM_E_ARG, "bst_softmax: null pointer");
  // the register kernel loads up to 16 bytes per lane (uint4 of 16-bit data at bs 32/64), the staged one bulk-copies
  if (((uintptr_t)x | (uintptr_t)y) & 15) return fail(BSMM_E_ARG, "bst_softmax: x and y must be 16-byte aligned");
  if ((long long)max_lut * bsize > 32768) return fail(BSMM_E_LIMIT, "bst_softmax: max_lut*bsize > 32768 (bst_op.cc:383)");
  if (autoregress_at_key >= 0 && (!mask || !nt_lut))
    return fail(BSMM_E_ARG, "bst_softmax: autoregress_at_key needs a mask and nt_lut");
  if (mask && mask_heads != 1 && mask_heads != heads) return fail(BSMM_E_ARG, "bst_softmax: mask_heads must be 1 or heads");
  cudaStream_t s = (cudaStream_t)stream;
  SoftmaxParams p = {};
  p.nn_lut = nn_lut; p.nt_lut = nt_lut;
  p.nn_head_stride = lut_heads > 1 ? 2LL * (ctx_blks_q + blocks) : 0;
  p.nt_head_stride = lut_heads > 1 ? 2LL * blocks : 0;
  p.mask = mask; p.mask_head_stride = (mask && mask_heads > 1) ? (long long)blocks * bsize : 0;
  p.autoregress_at_key = autoregress_at_key;
  p.x = x; p.y = y; p.scale = scale;
  p.batch = batch; p.heads = heads; p.blocks = blocks; p.ctx_blks_q = ctx_blks_q;
  // TMA-staged kernel: 16-bit tensors, 32 x 32 / 64 x 64 blocks, every row's blocks fit shared memory (<= 16 of them)
  static const bool no_staged = [] { const char* e = getenv("BSMM_SOFTMAX_STAGED"); return e && atoi(e) == 0; }();
  if (!no_staged && x_dtype != BSMM_F32 && y_dtype != BSMM_F32 && (bsize == 32 || bsize == 64) && max_lut >= 1 && max_lut <= 16 &&
      device_info().ok && device_info().cc_major >= 9) {
#define BSMM_SM_STAGED(TXT, TYT)                                                                              \
    return bsize == 64 ? launch_softmax_staged<TXT, TYT, 64>(p, max_lut, s) : launch_softmax_staged<TXT, TYT, 32>(p, max_lut, s);
    if (x_dtype == BSMM_BF16 && y_dtype == BSMM_BF16) { BSMM_SM_STAGED(__nv_bfloat16, __nv_bfloat16) }
    if (x_dtype == BSMM_BF16 && y_dtype == BSMM_F16)  { BSMM_SM_STAGED(__nv_bfloat16, __half) }
    if (x_dtype == BSMM_F16 && y_dtype == BSMM_F16)   { BSMM_SM_STAGED(__half, __half) }
    if (x_dtype == BSMM_F16 && y_dtype == BSMM_BF16)  { BSMM_SM_STAGED(__half, __nv_bfloat16) }
#undef BSMM_SM_STAGED
  }
  BSMM_DISPATCH_DTYPE(x_dtype, TX, {
    BSMM_DISPATCH_DTYPE(y_dtype, TY, {
      BSMM_DISPATCH_BSIZE(bsize, BS, {
        const long long groups = (long long)ctx_blks_q * SoftmaxMap<BS>::GROUPS;
        dim3 grid((unsigned)((groups + SOFTMAX_WARPS - 1) / SOFTMAX_WARPS), heads, batch);
        bst_softmax_kernel<TX, TY, BS><<<grid, SOFTMAX_WARPS * 32, 0, s>>>(p);
      });
    });
  });
  return check_launch("bst_softmax");
}

int bst_softmax_grad(int dtype, int dx_dtype, int bsize,
                     const int32_t* nn_lut, int lut_heads, int blocks, int max_lut,
                     const void* dy, const void* y, void* dx, float scale,
                     int batch, int heads, int ctx_blks_q, void* stream) {
  if (int e = check_bst(bsize, lut_heads, heads, 8, batch, blocks)) return e;
  if (!nn_lut || !dy || !y || !dx) return fail(BSMM_E_ARG, "bst_softmax_grad: null pointer");
  if (((uintptr_t)dy | (uintptr_t)y | (uintptr_t)dx) & 15)
    return fail(BSMM_E_ARG, "bst_softmax_grad: dy, y and dx must be 16-byte aligned");
  if ((long long)max_lut * bsize > 32768) return fail(BSMM_E_LIMIT, "bst_softmax_grad: max_lut*bsize > 32768");
  cudaStream_t s = (cudaStream_t)stream;
  SoftmaxParams p = {};
  p.nn_lut = nn_lut;
  p.nn_head_stride = lut_heads > 1 ? 2LL * (ctx_blks_q + blocks) : 0;
  p.x = dy; p.y_in = y; p.y = dx; p.scale = scale;
  p.batch = batch; p.heads = heads; p.blocks = blocks; p.ctx_blks_q = ctx_blks_q;
  static const bool no_staged = [] { const char* e = getenv("BSMM_SOFTMAX_STAGED"); return e && atoi(e) == 0; }();
  if (!no_staged && dtype != BSMM_F32 && dx_dtype != BSMM_F32 && (bsize == 32 || bsize == 64) && max_lut >= 1 && max_lut <= 16 &&
      device_info().ok && device_info().cc_major >= 9) {
#define BSMM_SG_STAGED(TT, TDT)                                                                               \
    return bsize == 64 ? launch_softmax_grad_staged<TT, TDT, 64>(p, max_lut, s) : launch_softmax_grad_staged<TT, TDT, 32>(p, max_lut, s);
    if (dtype == BSMM_BF16 && dx_dtype == BSMM_BF16) { BSMM_SG_STAGED(__nv_bfloat16, __nv_bfloat16) }
    if (dtype == BSMM_F16 && dx_dtype == BSMM_F16)   { BSMM_SG_STAGED(__half, __half) }
    if (dtype == BSMM_F16 && dx_dtype == BSMM_BF16)  { BSMM_SG_STAGED(__half, __nv_bfloat16) }
    if (dtype == BSMM_BF16 && dx_dtype == BSMM_F16)  { BSMM_SG_STAGED(__nv_bfloat16, __half) }
#undef BSMM_SG_STAGED
  }
  BSMM_DISPATCH_DTYPE(dtype, T, {
    BSMM_DISPATCH_DTYPE(dx_dtype, TD, {
      BSMM_DISPATCH_BSIZE(bsize, BS, {
        const long long groups = (long long)ctx_blks_q * SoftmaxMap<BS>::GROUPS;
        dim3 grid((unsigned)((groups + SOFTMAX_WARPS - 1) / SOFTMAX_WARPS), heads, batch);
        bst_softmax_grad_kernel<T, TD, BS><<<grid, SOFTMAX_WARPS * 32, 0, s>>>(p);
      });
    });
  });
  return check_launch("bst_softmax_grad");
}

int bst_attention(int dtype, int bsize, const int32_t* nn_lut, int lut_heads, int blocks,
                  const void* mask, int mask_heads, int autoregress_at_key,
                  const void* q, const void* k, const void* v, void* o, float scale,
                  int batch, int heads, int head_state, int ctx_blks_q, int ctx_blks_k, void* stream) {
  if (int e = check_bst(bsize, lut_heads, heads, head_state, batch, blocks)) return e;
  if (!nn_lut || !q || !k || !v || !o) return fail(BSMM_E_ARG, "bst_attention: null pointer");
  if (ctx_blks_q <= 0 || ctx_blks_k <= 0) return fail(BSMM_E_ARG, "bst_attention: bad context sizes");
  if (autoregress_at_key >= 0 && !mask) return fail(BSMM_E_ARG, "bst_attention: autoregress_at_key needs a mask");
  if (mask && mask_heads != 1 && mask_heads != heads) return fail(BSMM_E_ARG, "bst_attention: mask_heads must be 1 or heads");
  // the fused kernel's envelope; the reason stays in bsmm_last_error()
  const int rc = tc_bst_attention(dtype, bsize, nn_lut, lut_heads, blocks, mask, mask_heads, autoregress_at_key, q, k, v, o,
                                  scale, batch, heads, head_state, ctx_blks_q, ctx_blks_k, (cudaStream_t)stream);
  return rc == TC_NOT_APPLICABLE ? BSMM_E_NOKERNEL : rc;
}

int bst_attention_train(int dtype, int bsize, const int32_t* nn_lut, int lut_heads, int blocks,
                        const void* mask, int mask_heads, int autoregress_at_key,
                        const void* q, const void* k, const void* v, void* o, float* row_max, float* row_sum, float scale,
                        int batch, int heads, int head_state, int ctx_blks_q, int ctx_blks_k, void* stream) {
  if (int e = check_bst(bsize, lut_heads, heads, head_state, batch, blocks)) return e;
  if (!nn_lut || !q || !k || !v || !o || !row_max || !row_sum) return fail(BSMM_E_ARG, "bst_attention_train: null pointer");
  if (ctx_blks_q <= 0 || ctx_blks_k <= 0) return fail(BSMM_E_ARG, "bst_attention_train: bad context sizes");
  if (autoregress_at_key >= 0 && !mask) return fail(BSMM_E_ARG, "bst_attention_train: autoregress_at_key needs a mask");
  if (mask && mask_heads != 1 && mask_heads != heads) return fail(BSMM_E_ARG, "bst_attention_train: mask_heads must be 1 or heads");
  const int rc = tc_bst_attention(dtype, bsize, nn_lut, lut_heads, blocks, mask, mask_heads, autoregress_at_key, q, k, v, o,
                                  scale, batch, heads, head_state, ctx_blks_q, ctx_blks_k, (cudaStream_t)stream, row_max, row_sum);
  return rc == TC_NOT_APPLICABLE ? BSMM_E_NOKERNEL : rc;
}

int bst_attention_grad(int dtype, int bsize, const int32_t* nn_lut, const int32_t* tn_lut, const int32_t* tn_order,
                       int lut_heads, int blocks, const void* mask, int mask_heads, int autoregress_at_key,
                       const void* q, const void* k, const void* v, const void* o, const void* dy,
                       const float* row_max, const float* row_sum, float* delta, void* dq, void* dk, void* dv, float scale,
                       int batch, int heads, int head_state, int ctx_blks_q, int ctx_blks_k, void* stream) {
  if (int e = check_bst(bsize, lut_heads, heads, head_state, batch, blocks)) return e;
  if (!nn_lut || !tn_lut || !tn_order || !q || !k || !v || !o || !dy || !row_max || !row_sum || !delta || !dq || !dk || !dv)
    return fail(BSMM_E_ARG, "bst_attention_grad: null pointer");
  if (ctx_blks_q <= 0 || ctx_blks_k <= 0) return fail(BSMM_E_ARG, "bst_attention_grad: bad context sizes");
  if (autoregress_at_key >= 0 && !mask) return fail(BSMM_E_ARG, "bst_attention_grad: autoregress_at_key needs a mask");
  if (mask && mask_heads != 1 && mask_heads != heads) return fail(BSMM_E_ARG, "bst_attention_grad: mask_heads must be 1 or heads");
  const int rc = tc_bst_attention_grad(dtype, bsize, nn_lut, tn_lut, tn_order, lut_heads, blocks, mask, mask_heads,
                                       autoregress_at_key, q, k, v, o, dy, row_max, row_sum, delta, dq, dk, dv, scale, batch,
                                       heads, head_state, ctx_blks_q, ctx_blks_k, (cudaStream_t)stream);
  return rc == TC_NOT_APPLICABLE ? BSMM_E_NOKERNEL : rc;
}

// The dropout entries: keep_prob 1 runs the counterpart's kernels, keep_prob in (0, 1) their DROP instantiations.
static int check_attention_dropout(const char* op, double keep_prob, const int64_t* seed_call, BstAttnDrop& drop) {
  if (!(keep_prob > 0.0 && keep_prob <= 1.0)) return fail(BSMM_E_ARG, "%s: keep_prob must be in (0, 1]", op);
  if (keep_prob < 1.0 && !seed_call) return fail(BSMM_E_ARG, "%s: null seed_call", op);
  drop.keep_prob = keep_prob;
  drop.seed_call = reinterpret_cast<const long long*>(seed_call);
  return 0;
}

int bst_attention_dropout(int dtype, int bsize, const int32_t* nn_lut, int lut_heads, int blocks,
                          const void* mask, int mask_heads, int autoregress_at_key,
                          const void* q, const void* k, const void* v, void* o, float scale,
                          int batch, int heads, int head_state, int ctx_blks_q, int ctx_blks_k,
                          double keep_prob, const int64_t* seed_call, void* stream) {
  BstAttnDrop drop;
  if (int e = check_attention_dropout("bst_attention_dropout", keep_prob, seed_call, drop)) return e;
  if (int e = check_bst(bsize, lut_heads, heads, head_state, batch, blocks)) return e;
  if (!nn_lut || !q || !k || !v || !o) return fail(BSMM_E_ARG, "bst_attention_dropout: null pointer");
  if (ctx_blks_q <= 0 || ctx_blks_k <= 0) return fail(BSMM_E_ARG, "bst_attention_dropout: bad context sizes");
  if (autoregress_at_key >= 0 && !mask) return fail(BSMM_E_ARG, "bst_attention_dropout: autoregress_at_key needs a mask");
  if (mask && mask_heads != 1 && mask_heads != heads) return fail(BSMM_E_ARG, "bst_attention_dropout: mask_heads must be 1 or heads");
  const int rc = tc_bst_attention(dtype, bsize, nn_lut, lut_heads, blocks, mask, mask_heads, autoregress_at_key, q, k, v, o,
                                  scale, batch, heads, head_state, ctx_blks_q, ctx_blks_k, (cudaStream_t)stream, nullptr,
                                  nullptr, keep_prob < 1.0 ? &drop : nullptr);
  return rc == TC_NOT_APPLICABLE ? BSMM_E_NOKERNEL : rc;
}

int bst_attention_train_dropout(int dtype, int bsize, const int32_t* nn_lut, int lut_heads, int blocks,
                                const void* mask, int mask_heads, int autoregress_at_key,
                                const void* q, const void* k, const void* v, void* o, float* row_max, float* row_sum,
                                float scale, int batch, int heads, int head_state, int ctx_blks_q, int ctx_blks_k,
                                double keep_prob, const int64_t* seed_call, void* stream) {
  BstAttnDrop drop;
  if (int e = check_attention_dropout("bst_attention_train_dropout", keep_prob, seed_call, drop)) return e;
  if (int e = check_bst(bsize, lut_heads, heads, head_state, batch, blocks)) return e;
  if (!nn_lut || !q || !k || !v || !o || !row_max || !row_sum)
    return fail(BSMM_E_ARG, "bst_attention_train_dropout: null pointer");
  if (ctx_blks_q <= 0 || ctx_blks_k <= 0) return fail(BSMM_E_ARG, "bst_attention_train_dropout: bad context sizes");
  if (autoregress_at_key >= 0 && !mask)
    return fail(BSMM_E_ARG, "bst_attention_train_dropout: autoregress_at_key needs a mask");
  if (mask && mask_heads != 1 && mask_heads != heads)
    return fail(BSMM_E_ARG, "bst_attention_train_dropout: mask_heads must be 1 or heads");
  const int rc = tc_bst_attention(dtype, bsize, nn_lut, lut_heads, blocks, mask, mask_heads, autoregress_at_key, q, k, v, o,
                                  scale, batch, heads, head_state, ctx_blks_q, ctx_blks_k, (cudaStream_t)stream, row_max,
                                  row_sum, keep_prob < 1.0 ? &drop : nullptr);
  return rc == TC_NOT_APPLICABLE ? BSMM_E_NOKERNEL : rc;
}

int bst_attention_grad_dropout(int dtype, int bsize, const int32_t* nn_lut, const int32_t* tn_lut, const int32_t* tn_order,
                               int lut_heads, int blocks, const void* mask, int mask_heads, int autoregress_at_key,
                               const void* q, const void* k, const void* v, const void* o, const void* dy,
                               const float* row_max, const float* row_sum, float* delta, void* dq, void* dk, void* dv,
                               float scale, int batch, int heads, int head_state, int ctx_blks_q, int ctx_blks_k,
                               double keep_prob, const int64_t* seed_call, void* stream) {
  BstAttnDrop drop;
  if (int e = check_attention_dropout("bst_attention_grad_dropout", keep_prob, seed_call, drop)) return e;
  if (int e = check_bst(bsize, lut_heads, heads, head_state, batch, blocks)) return e;
  if (!nn_lut || !tn_lut || !tn_order || !q || !k || !v || !o || !dy || !row_max || !row_sum || !delta || !dq || !dk || !dv)
    return fail(BSMM_E_ARG, "bst_attention_grad_dropout: null pointer");
  if (ctx_blks_q <= 0 || ctx_blks_k <= 0) return fail(BSMM_E_ARG, "bst_attention_grad_dropout: bad context sizes");
  if (autoregress_at_key >= 0 && !mask)
    return fail(BSMM_E_ARG, "bst_attention_grad_dropout: autoregress_at_key needs a mask");
  if (mask && mask_heads != 1 && mask_heads != heads)
    return fail(BSMM_E_ARG, "bst_attention_grad_dropout: mask_heads must be 1 or heads");
  const int rc = tc_bst_attention_grad(dtype, bsize, nn_lut, tn_lut, tn_order, lut_heads, blocks, mask, mask_heads,
                                       autoregress_at_key, q, k, v, o, dy, row_max, row_sum, delta, dq, dk, dv, scale, batch,
                                       heads, head_state, ctx_blks_q, ctx_blks_k, (cudaStream_t)stream,
                                       keep_prob < 1.0 ? &drop : nullptr);
  return rc == TC_NOT_APPLICABLE ? BSMM_E_NOKERNEL : rc;
}

// The grouped-query entries: kv_heads divides heads; then the counterpart's checks and envelope, on kv-head-sized k, v.
static int check_kv_heads(const char* op, int heads, int kv_heads) {
  if (kv_heads < 1 || kv_heads > heads || heads % kv_heads)
    return fail(BSMM_E_ARG, "%s: kv_heads must divide heads and lie in [1, heads], got kv_heads %d, heads %d", op,
                kv_heads, heads);
  return 0;
}

int bst_attention_gqa(int dtype, int bsize, const int32_t* nn_lut, int lut_heads, int blocks,
                      const void* mask, int mask_heads, int autoregress_at_key,
                      const void* q, const void* k, const void* v, void* o, float scale,
                      int batch, int heads, int kv_heads, int head_state, int ctx_blks_q, int ctx_blks_k,
                      double keep_prob, const int64_t* seed_call, void* stream) {
  const char* what = "bst_attention_gqa";
  BstAttnDrop drop;
  if (int e = check_attention_dropout(what, keep_prob, seed_call, drop)) return e;
  if (int e = check_bst(bsize, lut_heads, heads, head_state, batch, blocks)) return e;
  if (int e = check_kv_heads(what, heads, kv_heads)) return e;
  if (!nn_lut || !q || !k || !v || !o) return fail(BSMM_E_ARG, "%s: null pointer", what);
  if (ctx_blks_q <= 0 || ctx_blks_k <= 0) return fail(BSMM_E_ARG, "%s: bad context sizes", what);
  if (autoregress_at_key >= 0 && !mask) return fail(BSMM_E_ARG, "%s: autoregress_at_key needs a mask", what);
  if (mask && mask_heads != 1 && mask_heads != heads) return fail(BSMM_E_ARG, "%s: mask_heads must be 1 or heads", what);
  const int rc = tc_bst_attention(dtype, bsize, nn_lut, lut_heads, blocks, mask, mask_heads, autoregress_at_key, q, k, v, o,
                                  scale, batch, heads, head_state, ctx_blks_q, ctx_blks_k, (cudaStream_t)stream, nullptr,
                                  nullptr, keep_prob < 1.0 ? &drop : nullptr, kv_heads);
  return rc == TC_NOT_APPLICABLE ? BSMM_E_NOKERNEL : rc;
}

int bst_attention_train_gqa(int dtype, int bsize, const int32_t* nn_lut, int lut_heads, int blocks,
                            const void* mask, int mask_heads, int autoregress_at_key,
                            const void* q, const void* k, const void* v, void* o, float* row_max, float* row_sum,
                            float scale, int batch, int heads, int kv_heads, int head_state, int ctx_blks_q,
                            int ctx_blks_k, double keep_prob, const int64_t* seed_call, void* stream) {
  const char* what = "bst_attention_train_gqa";
  BstAttnDrop drop;
  if (int e = check_attention_dropout(what, keep_prob, seed_call, drop)) return e;
  if (int e = check_bst(bsize, lut_heads, heads, head_state, batch, blocks)) return e;
  if (int e = check_kv_heads(what, heads, kv_heads)) return e;
  if (!nn_lut || !q || !k || !v || !o || !row_max || !row_sum) return fail(BSMM_E_ARG, "%s: null pointer", what);
  if (ctx_blks_q <= 0 || ctx_blks_k <= 0) return fail(BSMM_E_ARG, "%s: bad context sizes", what);
  if (autoregress_at_key >= 0 && !mask) return fail(BSMM_E_ARG, "%s: autoregress_at_key needs a mask", what);
  if (mask && mask_heads != 1 && mask_heads != heads) return fail(BSMM_E_ARG, "%s: mask_heads must be 1 or heads", what);
  const int rc = tc_bst_attention(dtype, bsize, nn_lut, lut_heads, blocks, mask, mask_heads, autoregress_at_key, q, k, v, o,
                                  scale, batch, heads, head_state, ctx_blks_q, ctx_blks_k, (cudaStream_t)stream, row_max,
                                  row_sum, keep_prob < 1.0 ? &drop : nullptr, kv_heads);
  return rc == TC_NOT_APPLICABLE ? BSMM_E_NOKERNEL : rc;
}

int bst_attention_grad_gqa(int dtype, int bsize, const int32_t* nn_lut, const int32_t* tn_lut, const int32_t* tn_order,
                           int lut_heads, int blocks, const void* mask, int mask_heads, int autoregress_at_key,
                           const void* q, const void* k, const void* v, const void* o, const void* dy,
                           const float* row_max, const float* row_sum, float* delta, void* dq, void* dk, void* dv,
                           float scale, int batch, int heads, int kv_heads, int head_state, int ctx_blks_q,
                           int ctx_blks_k, double keep_prob, const int64_t* seed_call, void* stream) {
  const char* what = "bst_attention_grad_gqa";
  BstAttnDrop drop;
  if (int e = check_attention_dropout(what, keep_prob, seed_call, drop)) return e;
  if (int e = check_bst(bsize, lut_heads, heads, head_state, batch, blocks)) return e;
  if (int e = check_kv_heads(what, heads, kv_heads)) return e;
  if (!nn_lut || !tn_lut || !tn_order || !q || !k || !v || !o || !dy || !row_max || !row_sum || !delta || !dq || !dk || !dv)
    return fail(BSMM_E_ARG, "%s: null pointer", what);
  if (ctx_blks_q <= 0 || ctx_blks_k <= 0) return fail(BSMM_E_ARG, "%s: bad context sizes", what);
  if (autoregress_at_key >= 0 && !mask) return fail(BSMM_E_ARG, "%s: autoregress_at_key needs a mask", what);
  if (mask && mask_heads != 1 && mask_heads != heads) return fail(BSMM_E_ARG, "%s: mask_heads must be 1 or heads", what);
  const int rc = tc_bst_attention_grad(dtype, bsize, nn_lut, tn_lut, tn_order, lut_heads, blocks, mask, mask_heads,
                                       autoregress_at_key, q, k, v, o, dy, row_max, row_sum, delta, dq, dk, dv, scale, batch,
                                       heads, head_state, ctx_blks_q, ctx_blks_k, (cudaStream_t)stream,
                                       keep_prob < 1.0 ? &drop : nullptr, kv_heads);
  return rc == TC_NOT_APPLICABLE ? BSMM_E_NOKERNEL : rc;
}

// ---- attention decode ---------------------------------------------------------------------------------------------
static bool decode_shape_ok(int bsize, int nn_max, int batch, int heads, int head_state, int n) {
  return (bsize == 16 || bsize == 32 || bsize == 64) && n >= 1 && n <= bsize && head_state > 0 && head_state % 16 == 0 &&
         head_state <= 256 && nn_max >= 0 && batch > 0 && heads > 0;
}

size_t bst_attention_decode_workspace_bytes(int bsize, int nn_max, int batch, int heads, int head_state, int n) {
  if (!decode_shape_ok(bsize, nn_max, batch, heads, head_state, n)) return 0;
  return bst_decode_workspace(nn_max, batch, heads, head_state, n);
}

static int attention_decode(const char* what, int dtype, int bsize, const int32_t* nn_lut, int lut_heads, int blocks,
                            int nn_max, const void* mask, int mask_heads, int autoregress_at_key, const void* q,
                            const void* k_cache, const void* v_cache, void* o, const int32_t* positions, int n,
                            float scale, int batch, int heads, int kv_heads, int head_state, int ctx_blks_q,
                            int ctx_blks_k, void* workspace, void* stream);

int bst_attention_decode(int dtype, int bsize, const int32_t* nn_lut, int lut_heads, int blocks, int nn_max,
                         const void* mask, int mask_heads, int autoregress_at_key,
                         const void* q, const void* k_cache, const void* v_cache, void* o,
                         const int32_t* positions, int n, float scale,
                         int batch, int heads, int head_state, int ctx_blks_q, int ctx_blks_k,
                         void* workspace, void* stream) {
  return attention_decode("bst_attention_decode", dtype, bsize, nn_lut, lut_heads, blocks, nn_max, mask, mask_heads,
                          autoregress_at_key, q, k_cache, v_cache, o, positions, n, scale, batch, heads, heads,
                          head_state, ctx_blks_q, ctx_blks_k, workspace, stream);
}

int bst_attention_decode_gqa(int dtype, int bsize, const int32_t* nn_lut, int lut_heads, int blocks, int nn_max,
                             const void* mask, int mask_heads, int autoregress_at_key,
                             const void* q, const void* k_cache, const void* v_cache, void* o,
                             const int32_t* positions, int n, float scale,
                             int batch, int heads, int kv_heads, int head_state, int ctx_blks_q, int ctx_blks_k,
                             void* workspace, void* stream) {
  const char* what = "bst_attention_decode_gqa";
  if (heads > 0 && check_kv_heads(what, heads, kv_heads)) return BSMM_E_ARG;
  return attention_decode(what, dtype, bsize, nn_lut, lut_heads, blocks, nn_max, mask, mask_heads, autoregress_at_key, q,
                          k_cache, v_cache, o, positions, n, scale, batch, heads, kv_heads, head_state, ctx_blks_q,
                          ctx_blks_k, workspace, stream);
}

// bst_attention_decode(_gqa) after the kv_heads check
static int attention_decode(const char* what, int dtype, int bsize, const int32_t* nn_lut, int lut_heads, int blocks,
                            int nn_max, const void* mask, int mask_heads, int autoregress_at_key, const void* q,
                            const void* k_cache, const void* v_cache, void* o, const int32_t* positions, int n,
                            float scale, int batch, int heads, int kv_heads, int head_state, int ctx_blks_q,
                            int ctx_blks_k, void* workspace, void* stream) {
  if (dtype != BSMM_F16 && dtype != BSMM_BF16)
    return fail(BSMM_E_DTYPE, "%s: fp16 or bf16 only (one dtype for q and both caches), got %d", what, dtype);
  if (bsize != 16 && bsize != 32 && bsize != 64) return fail(BSMM_E_BSIZE, "%s: block size must be 16, 32 or 64, got %d", what, bsize);
  if (n < 1 || n > bsize) return fail(BSMM_E_ARG, "%s: n must be in [1, block size %d], got %d", what, bsize, n);
  if (head_state <= 0 || head_state % 16 || head_state > 256)
    return fail(BSMM_E_ARG, "%s: head_state must be a multiple of 16 up to 256, got %d", what, head_state);
  if (batch <= 0 || heads <= 0 || blocks <= 0 || nn_max < 0 || ctx_blks_q <= 0 || ctx_blks_k <= 0)
    return fail(BSMM_E_ARG, "%s: bad batch / heads / blocks / nn_max / context sizes", what);
  if (lut_heads != 1 && lut_heads != heads) return fail(BSMM_E_ARG, "%s: lut_heads must be 1 or heads", what);
  if (mask && mask_heads != 1 && mask_heads != heads) return fail(BSMM_E_ARG, "%s: mask_heads must be 1 or heads", what);
  if (autoregress_at_key >= 0 && !mask) return fail(BSMM_E_ARG, "%s: autoregress_at_key needs a mask", what);
  if (!nn_lut || !q || !k_cache || !v_cache || !o || !positions) return fail(BSMM_E_ARG, "%s: null pointer", what);
  if (((uintptr_t)q | (uintptr_t)k_cache | (uintptr_t)v_cache | (uintptr_t)o) & 15)
    return fail(BSMM_E_ARG, "%s: q, the caches and o must be 16-byte aligned", what);
  const size_t ws = bst_decode_workspace(nn_max, batch, heads, head_state, n);
  if (ws > 0 && !workspace)
    return fail(BSMM_E_ARG, "%s: null workspace (bst_attention_decode_workspace_bytes gives its size)", what);
  if ((uintptr_t)workspace & 15) return fail(BSMM_E_ARG, "%s: the workspace must be 16-byte aligned", what);
  if ((long long)batch * heads * 2 * bst_decode_nsplit(nn_max) >= (1LL << 31) || (long long)batch * n * heads >= (1LL << 31))
    return fail(BSMM_E_LIMIT, "%s: too many CTAs for one grid", what);
  if (!wgmma_device()) return fail(BSMM_E_NODEV, "%s: needs an sm_90 device", what);
  return tc_bst_attention_decode(dtype, bsize, nn_lut, lut_heads, blocks, nn_max, mask, mask_heads, autoregress_at_key,
                                 q, k_cache, v_cache, o, positions, n, scale, batch, heads, head_state, ctx_blks_q,
                                 ctx_blks_k, workspace, (cudaStream_t)stream, kv_heads);
}

int bst_autoregressive_mask(int bsize, const int32_t* nt_lut, int lut_heads, int blocks,
                            const void* mask_in, void* mask_out, int autoregress_at_key, void* stream) {
  if (!nt_lut || !mask_in || !mask_out || lut_heads <= 0 || blocks <= 0)
    return fail(BSMM_E_ARG, "bst_autoregressive_mask: bad arguments");
  cudaStream_t s = (cudaStream_t)stream;
  dim3 grid((blocks * bsize + 127) / 128, lut_heads);
  BSMM_DISPATCH_BSIZE(bsize, BS, {
    bst_autoregressive_mask_kernel<BS><<<grid, 128, 0, s>>>(nt_lut, lut_heads > 1 ? 2LL * blocks : 0,
                                                            mask_in, mask_out, blocks, autoregress_at_key);
  });
  return check_launch("bst_autoregressive_mask");
}

// ---- dense softmax and top-k (csrc/dense_softmax.cuh) ---------------------------------------------------------------
static bool dense_dtype_ok(int dtype) { return dtype == BSMM_F32 || dtype == BSMM_F16 || dtype == BSMM_BF16; }

// Validates the (D0, D1, D2, D3) shape and the mask strides, fills a's row map; `rows` = 0 means nothing to launch.
static int dense_args(const char* what, int dtype, long long D0, int D1, int D2, int D3, const float* mask,
                      long long M1, long long M2, DenseArgs& a) {
  if (!dense_dtype_ok(dtype)) return fail(BSMM_E_ARG, "%s: unsupported dtype code %d", what, dtype);
  if (D0 < 0 || D1 < 0 || D2 < 0 || D3 <= 0) return fail(BSMM_E_ARG, "%s: bad sizes (%lld, %d, %d, %d)", what, D0, D1, D2, D3);
  if (!mask) M1 = M2 = 0;
  if ((M2 != 0 && M2 != D3) || (M1 != 0 && M1 != (long long)D3 * (M2 ? D2 : 1)))
    return fail(BSMM_E_ARG, "%s: mask strides (%lld, %lld) do not describe a (1|D1, 1|D2, D3) mask", what, M1, M2);
  a.mask = mask;
  a.D3 = D3;
  a.rows = D0 * D1 * D2;
  a.map = {D1, D2, M1, M2, D0 * (M1 ? 1 : D1) * (M2 ? 1 : D2)};
  // one CTA per row on every route but the warp one; grid.x holds at most 2^31 - 1
  if (a.rows > 0x7fffffffLL * (D3 <= DSM_WARP_MAX ? DSM_WARPS : 1))
    return fail(BSMM_E_LIMIT, "%s: %lld rows exceed the grid", what, a.rows);
  return 0;
}

static bool aligned16(const void* p) { return ((uintptr_t)p & 15) == 0; }

int bst_dense_softmax(int dtype, const void* x, const float* mask, void* y, long long D0, int D1, int D2, int D3,
                      long long mask_stride1, long long mask_stride2, float scale, void* stream) {
  DenseArgs a = {};
  if (int e = dense_args("bst_dense_softmax", dtype, D0, D1, D2, D3, mask, mask_stride1, mask_stride2, a)) return e;
  if (!x || !y) return fail(BSMM_E_ARG, "bst_dense_softmax: null pointer");
  if (a.rows == 0) return 0;
  a.a = x; a.out = y; a.scale = scale;
  const bool vec = aligned16(x) && aligned16(y) && (!mask || aligned16(mask)) && D3 % (16 / dtype_size(dtype)) == 0;
  BSMM_DISPATCH_DTYPE(dtype, T, { return launch_dense_softmax<T>(a, false, vec, (cudaStream_t)stream); });
  return 0;
}

int bst_dense_softmax_grad(int dtype, const void* dy, const void* y, const float* mask, void* dx, long long D0, int D1,
                           int D2, int D3, long long mask_stride1, long long mask_stride2, float scale, void* stream) {
  DenseArgs a = {};
  if (int e = dense_args("bst_dense_softmax_grad", dtype, D0, D1, D2, D3, mask, mask_stride1, mask_stride2, a)) return e;
  if (!dy || !y || !dx) return fail(BSMM_E_ARG, "bst_dense_softmax_grad: null pointer");
  if (a.rows == 0) return 0;
  a.a = dy; a.b = y; a.out = dx; a.scale = scale;
  const bool vec = aligned16(dy) && aligned16(y) && aligned16(dx) && (!mask || aligned16(mask)) &&
                   D3 % (16 / dtype_size(dtype)) == 0;
  BSMM_DISPATCH_DTYPE(dtype, T, { return launch_dense_softmax<T>(a, true, vec, (cudaStream_t)stream); });
  return 0;
}

int bst_topk_softmax(int dtype, const void* x, const float* mask, void* y, long long D0, int D1, int D2, int D3,
                     long long mask_stride1, long long mask_stride2, int k, float scale, void* stream) {
  DenseArgs a = {};
  if (int e = dense_args("bst_topk_softmax", dtype, D0, D1, D2, D3, mask, mask_stride1, mask_stride2, a)) return e;
  if (!x || !y) return fail(BSMM_E_ARG, "bst_topk_softmax: null pointer");
  if (D3 > TOPK_MAX || k < 1 || k > D3) return fail(BSMM_E_ARG, "bst_topk_softmax: need 1 <= k <= D3 <= %d, got k %d, D3 %d", TOPK_MAX, k, D3);
  if (a.rows > 0x7fffffffLL) return fail(BSMM_E_LIMIT, "bst_topk_softmax: %lld rows exceed the grid", a.rows);
  if (a.rows == 0) return 0;
  a.a = x; a.out = y; a.k = k; a.mode = TOPK_SOFTMAX; a.scale = scale;
  BSMM_DISPATCH_DTYPE(dtype, T, { return launch_dense_topk<T>(a, (cudaStream_t)stream); });
  return 0;
}

// ---- softmax cross entropy (csrc/dense_softmax.cuh) and transpose (csrc/transpose.cuh) -------------------------------
static int xent_args(const char* what, int dtype, int label_type, long long N, int K) {
  if (!dense_dtype_ok(dtype)) return fail(BSMM_E_ARG, "%s: unsupported dtype code %d", what, dtype);
  if (label_type < BSMM_LABEL_U8 || label_type > BSMM_LABEL_I64)
    return fail(BSMM_E_ARG, "%s: unsupported label type %d", what, label_type);
  if (N < 0 || K <= 0) return fail(BSMM_E_ARG, "%s: bad sizes N %lld, K %d", what, N, K);
  // one CTA per row on the CTA route; grid.x holds at most 2^31 - 1
  if (N > 0x7fffffffLL * (K <= DSM_WARP_MAX ? DSM_WARPS : 1)) return fail(BSMM_E_LIMIT, "%s: %lld rows exceed the grid", what, N);
  return 0;
}

int bst_softmax_xent(int dtype, int label_type, const void* logits, const void* labels, float* loss, float* lse,
                     long long N, int K, void* stream) {
  if (int e = xent_args("bst_softmax_xent", dtype, label_type, N, K)) return e;
  if (!logits || !labels || !loss || !lse) return fail(BSMM_E_ARG, "bst_softmax_xent: null pointer");
  if (N == 0) return 0;
  XentArgs a = {};
  a.x = logits; a.labels = labels; a.loss = loss; a.lse = lse; a.rows = N; a.K = K; a.label_type = label_type;
  const bool vec = aligned16(logits) && K % (16 / dtype_size(dtype)) == 0;
  BSMM_DISPATCH_DTYPE(dtype, T, { return launch_softmax_xent<T>(a, false, vec, (cudaStream_t)stream); });
  return 0;
}

int bst_softmax_xent_grad(int dtype, int label_type, const void* logits, const void* labels, const float* lse,
                          const float* dy, void* dx, long long N, int K, void* stream) {
  if (int e = xent_args("bst_softmax_xent_grad", dtype, label_type, N, K)) return e;
  if (!logits || !labels || !lse || !dy || !dx) return fail(BSMM_E_ARG, "bst_softmax_xent_grad: null pointer");
  if (N == 0) return 0;
  XentArgs a = {};
  a.x = logits; a.labels = labels; a.lse_in = lse; a.dy = dy; a.dx = dx; a.rows = N; a.K = K; a.label_type = label_type;
  const bool vec = aligned16(logits) && aligned16(dx) && K % (16 / dtype_size(dtype)) == 0;
  BSMM_DISPATCH_DTYPE(dtype, T, { return launch_softmax_xent<T>(a, true, vec, (cudaStream_t)stream); });
  return 0;
}

int bst_transpose_0213(int dtype, const void* x, void* y, long long D0, long long D1, long long D2, long long D3,
                       void* stream) {
  if (!dense_dtype_ok(dtype)) return fail(BSMM_E_ARG, "bst_transpose_0213: unsupported dtype code %d", dtype);
  if (D0 < 0 || D1 < 0 || D2 < 0 || D3 < 0)
    return fail(BSMM_E_ARG, "bst_transpose_0213: bad sizes (%lld, %lld, %lld, %lld)", D0, D1, D2, D3);
  if (!x || !y) return fail(BSMM_E_ARG, "bst_transpose_0213: null pointer");
  if (D0 == 0 || D1 == 0 || D2 == 0 || D3 == 0) return 0;
  if (D0 > LLONG_MAX / D1 / D2 / D3) return fail(BSMM_E_LIMIT, "bst_transpose_0213: more than 2^63 elements");
  return launch_transpose_0213(dtype_size(dtype), x, y, D0, D1, D2, D3, (cudaStream_t)stream);
}

int bst_topk(int dtype, const void* x, void* y, int32_t* idx, long long rows, int D3, int k, int mode, void* stream) {
  if (!dense_dtype_ok(dtype)) return fail(BSMM_E_ARG, "bst_topk: unsupported dtype code %d", dtype);
  if (mode < TOPK_VALUES || mode > TOPK_REBASE) return fail(BSMM_E_ARG, "bst_topk: mode must be 0, 1 or 2, got %d", mode);
  if (!x || !y || (mode == TOPK_VALUES && !idx)) return fail(BSMM_E_ARG, "bst_topk: null pointer");
  if (rows < 0 || D3 <= 0 || D3 > TOPK_MAX || k < 1 || k > D3)
    return fail(BSMM_E_ARG, "bst_topk: need rows >= 0 and 1 <= k <= D3 <= %d, got k %d, D3 %d", TOPK_MAX, k, D3);
  if (rows > 0x7fffffffLL) return fail(BSMM_E_LIMIT, "bst_topk: %lld rows exceed the grid", rows);
  if (rows == 0) return 0;
  DenseArgs a = {};
  a.a = x; a.out = y; a.idx = idx; a.D3 = D3; a.k = k; a.mode = mode; a.rows = rows;
  a.map = {1, 1, 0, 0, rows};
  BSMM_DISPATCH_DTYPE(dtype, T, { return launch_dense_topk<T>(a, (cudaStream_t)stream); });
  return 0;
}

// ---- layer norm (csrc/layer_norm.cuh) -------------------------------------------------------------------------------------
static int ln_args(const char* what, int dtype, int gdtype, int axis, long long N, int K, int segments, float epsilon) {
  if (!dense_dtype_ok(dtype) || !dense_dtype_ok(gdtype))
    return fail(BSMM_E_ARG, "%s: unsupported dtype codes %d, %d", what, dtype, gdtype);
  if (axis != 0 && axis != 1) return fail(BSMM_E_ARG, "%s: axis must be 0 or 1, got %d", what, axis);
  if (N < 0 || K <= 0 || segments <= 0 || K % segments)
    return fail(BSMM_E_ARG, "%s: bad sizes N %lld, K %d, segments %d", what, N, K, segments);
  if (axis == 0 && segments != 1) return fail(BSMM_E_ARG, "%s: segments need axis 1", what);
  if (!(epsilon >= 0.f)) return fail(BSMM_E_ARG, "%s: epsilon must be >= 0", what);
  const int L = K / segments;
  if (axis == 1 && N * segments > 0x7fffffffLL * (L <= DSM_WARP_MAX ? DSM_WARPS : 1))
    return fail(BSMM_E_LIMIT, "%s: %lld rows exceed the grid", what, N * segments);
  if (axis == 0 && (N > 0x7fffffffLL * 32 || K > 65535LL * LN_CN_MIN_ROWS))
    return fail(BSMM_E_LIMIT, "%s: N %lld or K %d exceeds the grid", what, N, K);
  return 0;
}

size_t bsmm_layer_norm_workspace_bytes(int axis, long long N, int K, int segments) {
  if ((axis != 0 && axis != 1) || N <= 0 || K <= 0 || segments <= 0 || K % segments) return 0;
  return ln_workspace_floats(axis, N, K, segments) * sizeof(float);
}

int bsmm_layer_norm(int dtype, int gdtype, int axis, const void* x, const void* g, const void* b, void* y, float* mean,
                    float* rstd, void* workspace, long long N, int K, int segments, float epsilon, int relu, void* stream) {
  if (int e = ln_args("bsmm_layer_norm", dtype, gdtype, axis, N, K, segments, epsilon)) return e;
  if (!x || !g || !b || !y || !mean || !rstd || (axis == 0 && !workspace)) return fail(BSMM_E_ARG, "bsmm_layer_norm: null pointer");
  if (N == 0) return 0;
  LnArgs a = {};
  a.x = x; a.g = g; a.b = b; a.gdtype = gdtype; a.y = y; a.mean = mean; a.rstd = rstd; a.ws = (float*)workspace;
  a.N = N; a.K = K; a.S = segments; a.L = K / segments; a.eps = epsilon; a.relu = relu != 0;
  const int V = 16 / dtype_size(dtype);
  if (axis == 0) {
    const bool vec = aligned16(x) && aligned16(y) && N % V == 0;
    BSMM_DISPATCH_DTYPE(dtype, T, { return launch_layer_norm_cn<T>(a, false, vec, gdtype, nullptr, nullptr, (cudaStream_t)stream); });
  } else {
    const bool vec = aligned16(x) && aligned16(y) && a.L % V == 0;
    BSMM_DISPATCH_DTYPE(dtype, T, { return launch_layer_norm_nc<T>(a, false, vec, gdtype, nullptr, nullptr, (cudaStream_t)stream); });
  }
  return 0;
}

int bsmm_layer_norm_grad(int dtype, int gdtype, int axis, const void* dy, const void* x, const void* g, const void* b,
                         const float* mean, const float* rstd, void* dx, void* dg, void* db, void* workspace, long long N,
                         int K, int segments, float epsilon, int relu, void* stream) {
  if (int e = ln_args("bsmm_layer_norm_grad", dtype, gdtype, axis, N, K, segments, epsilon)) return e;
  if (!dy || !x || !g || !b || !mean || !rstd || !dx || !dg || !db || !workspace)
    return fail(BSMM_E_ARG, "bsmm_layer_norm_grad: null pointer");
  if (N == 0) return 0;
  LnArgs a = {};
  a.x = x; a.dy = dy; a.g = g; a.b = b; a.gdtype = gdtype; a.y = dx; a.mean = (float*)mean; a.rstd = (float*)rstd;
  a.ws = (float*)workspace; a.N = N; a.K = K; a.S = segments; a.L = K / segments; a.eps = epsilon; a.relu = relu != 0;
  const int V = 16 / dtype_size(dtype);
  if (axis == 0) {
    const bool vec = aligned16(x) && aligned16(dy) && aligned16(dx) && N % V == 0;
    BSMM_DISPATCH_DTYPE(dtype, T, { return launch_layer_norm_cn<T>(a, true, vec, gdtype, dg, db, (cudaStream_t)stream); });
  } else {
    const bool vec = aligned16(x) && aligned16(dy) && aligned16(dx) && a.L % V == 0;
    BSMM_DISPATCH_DTYPE(dtype, T, { return launch_layer_norm_nc<T>(a, true, vec, gdtype, dg, db, (cudaStream_t)stream); });
  }
  return 0;
}

// ---- bias + activation and dropout (csrc/ewops.cuh) ------------------------------------------------------------------------
static int br_args(const char* what, int dtype, int bdtype, int axis, long long N, int K, int act) {
  if (!dense_dtype_ok(dtype) || !dense_dtype_ok(bdtype))
    return fail(BSMM_E_ARG, "%s: unsupported dtype codes %d, %d", what, dtype, bdtype);
  if (axis != 0 && axis != 1) return fail(BSMM_E_ARG, "%s: axis must be 0 or 1, got %d", what, axis);
  if (N < 0 || K <= 0) return fail(BSMM_E_ARG, "%s: bad sizes N %lld, K %d", what, N, K);
  if (act < ACT_NONE || act > ACT_FAST_GELU) return fail(BSMM_E_ARG, "%s: act must be 0, 1 or 2, got %d", what, act);
  if (axis == 0 && (N + BR_SEG - 1) / BR_SEG > 0x7fffffffLL) return fail(BSMM_E_LIMIT, "%s: N %lld exceeds the grid", what, N);
  return 0;
}

size_t bsmm_bias_grad_workspace_bytes(int axis, long long N, int K) {
  if ((axis != 0 && axis != 1) || N <= 0 || K <= 0) return 0;
  return br_workspace_floats(axis, N, K) * sizeof(float);
}

int bsmm_bias_relu(int dtype, int bdtype, int axis, const void* x, const void* b, void* y, long long N, int K, int act,
                   void* stream) {
  if (int e = br_args("bsmm_bias_relu", dtype, bdtype, axis, N, K, act)) return e;
  if (!x || !b || !y) return fail(BSMM_E_ARG, "bsmm_bias_relu: null pointer");
  if (N == 0) return 0;
  BrArgs a = {};
  a.x = x; a.b = b; a.y = y; a.N = N; a.K = K; a.bdt = bdtype; a.act = act;
  const bool vec = aligned16(x) && aligned16(y) && (axis ? K : N) % (16 / dtype_size(dtype)) == 0;
  BSMM_DISPATCH_DTYPE(dtype, T, { return launch_bias_act<T>(a, axis, false, vec, nullptr, (cudaStream_t)stream); });
  return 0;
}

int bsmm_bias_relu_grad(int dtype, int bdtype, int axis, const void* dy, const void* src, const void* b, void* dx,
                        void* db, void* workspace, long long N, int K, int act, void* stream) {
  if (int e = br_args("bsmm_bias_relu_grad", dtype, bdtype, axis, N, K, act)) return e;
  if (!dy || !b || !db || !workspace || (act != ACT_NONE && (!src || !dx)))
    return fail(BSMM_E_ARG, "bsmm_bias_relu_grad: null pointer");
  if (N == 0) return 0;
  BrArgs a = {};
  a.x = dy; a.src = src; a.b = b; a.y = dx; a.part = (float*)workspace; a.N = N; a.K = K; a.bdt = bdtype; a.act = act;
  const bool vec = aligned16(dy) && (act == ACT_NONE || (aligned16(src) && aligned16(dx))) &&
                   (axis ? K : N) % (16 / dtype_size(dtype)) == 0;
  BSMM_DISPATCH_DTYPE(dtype, T, { return launch_bias_act<T>(a, axis, true, vec, db, (cudaStream_t)stream); });
  return 0;
}

int bsmm_dropout_mask(int32_t* mask, long long M, double keep_prob, long long* state, void* stream) {
  if (!mask || !state) return fail(BSMM_E_ARG, "bsmm_dropout_mask: null pointer");
  if (M < 0) return fail(BSMM_E_ARG, "bsmm_dropout_mask: bad size %lld", M);
  if (!(keep_prob > 0.0 && keep_prob <= 1.0)) return fail(BSMM_E_ARG, "bsmm_dropout_mask: keep_prob must be in (0, 1]");
  if (M == 0) return 0;
  const unsigned long long thr = (unsigned long long)floor(keep_prob * 4294967296.0);
  return launch_dropout_mask((uint32_t*)mask, M, thr, state, (cudaStream_t)stream);
}

int bsmm_dropout_apply(int dtype, const void* x, const int32_t* mask, void* y, int ndim, const long long* shape,
                       const long long* mask_strides, long long mask_words, double keep_prob, void* stream) {
  if (!dense_dtype_ok(dtype)) return fail(BSMM_E_ARG, "bsmm_dropout_apply: unsupported dtype code %d", dtype);
  if (ndim < 0 || ndim > DROP_MAX_DIMS) return fail(BSMM_E_ARG, "bsmm_dropout_apply: ndim must be in [0, %d]", DROP_MAX_DIMS);
  if (ndim > 0 && (!shape || !mask_strides)) return fail(BSMM_E_ARG, "bsmm_dropout_apply: null shape or strides");
  if (!(keep_prob > 0.0 && keep_prob <= 1.0)) return fail(BSMM_E_ARG, "bsmm_dropout_apply: keep_prob must be in (0, 1]");
  DropArgs a = {};
  long long n = 1, top = 0;
  for (int d = 0; d < ndim; ++d) {
    if (shape[d] < 0 || mask_strides[d] < 0) return fail(BSMM_E_ARG, "bsmm_dropout_apply: negative size or stride in dim %d", d);
    if (shape[d] == 0) n = 0;
    else if (n && shape[d] > LLONG_MAX / n) return fail(BSMM_E_LIMIT, "bsmm_dropout_apply: more than 2^63 elements");
    else n *= shape[d];
  }
  if (!x || !mask || !y) return fail(BSMM_E_ARG, "bsmm_dropout_apply: null pointer");
  if (n == 0) return mask_words < 0 ? fail(BSMM_E_ARG, "bsmm_dropout_apply: bad mask_words") : 0;
  // drop size-1 dims; merge a dim into the next inner one when both broadcast or both are contiguous in the mask
  for (int d = 0; d < ndim; ++d) {
    if (shape[d] == 1) continue;
    top += (shape[d] - 1) * mask_strides[d];
    const long long st = mask_strides[d];
    if (a.nd > 0) {
      const int i = a.nd - 1;
      if ((a.mst[i] == 0 && st == 0) || (st != 0 && a.mst[i] == st * shape[d])) {
        a.size[i] *= shape[d];
        a.mst[i] = st;
        continue;
      }
    }
    a.size[a.nd] = shape[d];
    a.mst[a.nd++] = st;
  }
  if (top >= mask_words * 32 || mask_words < 1) return fail(BSMM_E_ARG, "bsmm_dropout_apply: the mask has too few words");
  if (a.nd > 0 && a.mst[a.nd - 1] > 1) return fail(BSMM_E_ARG, "bsmm_dropout_apply: the innermost mask stride must be 0 or 1");
  if (a.nd == 1 && a.mst[0] == 1) a.nd = 0;
  a.x = x; a.mask = (const uint32_t*)mask; a.y = y; a.n = n; a.words = mask_words; a.scale = (float)(1.0 / keep_prob);
  const int V = 16 / dtype_size(dtype);
  const bool vec = aligned16(x) && aligned16(y) && (a.nd == 0 ? n : a.size[a.nd - 1]) % V == 0;
  BSMM_DISPATCH_DTYPE(dtype, T, { return launch_dropout_apply<T>(a, vec, (cudaStream_t)stream); });
  return 0;
}

// ---- LSTM gates and sparse relu (csrc/lstm.cuh) ----------------------------------------------------------------------------
static int lstm_args(const char* what, int dtype, int bdtype, long long N, int K, long long stride) {
  if (!dense_dtype_ok(dtype) || !dense_dtype_ok(bdtype))
    return fail(BSMM_E_ARG, "%s: unsupported dtype codes %d, %d", what, dtype, bdtype);
  if (N < 0 || K <= 0 || stride < K) return fail(BSMM_E_ARG, "%s: bad sizes N %lld, K %d, stride %lld", what, N, K, stride);
  if (N > LLONG_MAX / stride) return fail(BSMM_E_LIMIT, "%s: more than 2^63 elements", what);
  return 0;
}

// 16-byte accesses when every pointer given is aligned and every row start stays so
static bool lstm_vec(int dtype, int K, long long stride, std::initializer_list<const void*> ptrs) {
  const int V = 16 / dtype_size(dtype);
  if (K % V || stride % V) return false;
  for (const void* p : ptrs)
    if (p && !aligned16(p)) return false;
  return true;
}

int bsmm_lstm_gates(int dtype, int bdtype, const void* c, const void* i, const void* u, const void* f, const void* o,
                    long long stride, const void* bias, void* c_next, void* h_next, long long N, int K,
                    float forget_bias, void* stream) {
  if (int e = lstm_args("bsmm_lstm_gates", dtype, bdtype, N, K, stride)) return e;
  if (!c || !i || !u || !f || !o || !c_next || !h_next) return fail(BSMM_E_ARG, "bsmm_lstm_gates: null pointer");
  if (N == 0) return 0;
  LstmArgs a = {};
  a.c = c; a.g[0] = i; a.g[1] = u; a.g[2] = f; a.g[3] = o; a.bias = bias; a.c_out = c_next; a.h_out = h_next;
  a.N = N; a.gs = stride; a.K = K; a.bdt = bdtype; a.forget_bias = forget_bias;
  const bool vec = lstm_vec(dtype, K, stride, {c, i, u, f, o, c_next, h_next});
  BSMM_DISPATCH_DTYPE(dtype, T, { return launch_lstm_gates<T>(a, false, vec, (cudaStream_t)stream); });
  return 0;
}

int bsmm_lstm_gates_grad(int dtype, int bdtype, const void* c, const void* i, const void* u, const void* f,
                         const void* o, long long stride, const void* bias, const void* ec, const void* eh, void* dc,
                         void* di, void* du, void* df, void* d_o, long long N, int K, float forget_bias, void* stream) {
  if (int e = lstm_args("bsmm_lstm_gates_grad", dtype, bdtype, N, K, stride)) return e;
  if (!c || !i || !u || !f || !o || !dc || !di || !du || !df || !d_o)
    return fail(BSMM_E_ARG, "bsmm_lstm_gates_grad: null pointer");
  if (N == 0) return 0;
  LstmArgs a = {};
  a.c = c; a.g[0] = i; a.g[1] = u; a.g[2] = f; a.g[3] = o; a.bias = bias; a.ec = ec; a.eh = eh; a.c_out = dc;
  a.dg[0] = di; a.dg[1] = du; a.dg[2] = df; a.dg[3] = d_o;
  a.N = N; a.gs = stride; a.K = K; a.bdt = bdtype; a.forget_bias = forget_bias;
  const bool vec = lstm_vec(dtype, K, stride, {c, i, u, f, o, ec, eh, dc, di, du, df, d_o});
  BSMM_DISPATCH_DTYPE(dtype, T, { return launch_lstm_gates<T>(a, true, vec, (cudaStream_t)stream); });
  return 0;
}

static int lstm_ln_args(const char* what, int dtype, int gdtype, long long N, int K, long long stride) {
  if (!dense_dtype_ok(dtype) || !dense_dtype_ok(gdtype))
    return fail(BSMM_E_ARG, "%s: unsupported dtype codes %d, %d", what, dtype, gdtype);
  if (N < 0 || K <= 0 || stride < 4LL * K)
    return fail(BSMM_E_ARG, "%s: bad sizes N %lld, K %d, stride %lld", what, N, K, stride);
  if (K > 0x7fffffff / 4) return fail(BSMM_E_LIMIT, "%s: 4K exceeds 2^31 - 1 (K %d)", what, K);
  if (N > LLONG_MAX / stride) return fail(BSMM_E_LIMIT, "%s: more than 2^63 elements", what);
  return 0;
}

size_t bsmm_lstm_ln_gates_workspace_bytes(long long N, int K) {
  if (N <= 0 || K <= 0 || K > 0x7fffffff / 4) return 0;
  int rpu, parts;
  lng_partition(N, rpu, parts);
  return (size_t)2 * parts * 4 * K * sizeof(float);
}

int bsmm_lstm_ln_gates(int dtype, int gdtype, const void* c, const void* z, long long stride, const void* g,
                       const void* b, void* c_next, void* h_next, float* mean, float* rstd, long long N, int K,
                       float epsilon, float forget_bias, void* stream) {
  if (int e = lstm_ln_args("bsmm_lstm_ln_gates", dtype, gdtype, N, K, stride)) return e;
  if (!(epsilon >= 0.f)) return fail(BSMM_E_ARG, "bsmm_lstm_ln_gates: epsilon must be >= 0");
  if (!c || !z || !g || !b || !c_next || !h_next || !mean || !rstd)
    return fail(BSMM_E_ARG, "bsmm_lstm_ln_gates: null pointer");
  if (N == 0) return 0;
  LnGatesArgs a = {};
  a.c = c; a.z = z; a.g = g; a.b = b; a.c_out = c_next; a.h_out = h_next; a.mean = mean; a.rstd = rstd;
  a.N = N; a.zs = stride; a.K = K; a.gdt = gdtype; a.eps = epsilon; a.forget_bias = forget_bias;
  BSMM_DISPATCH_DTYPE(dtype, T, { return launch_lstm_ln_gates<T>(a, false, (cudaStream_t)stream); });
  return 0;
}

int bsmm_lstm_ln_gates_grad(int dtype, int gdtype, const void* c, const void* z, long long stride, const void* g,
                            const void* b, const float* mean, const float* rstd, const void* ec, const void* eh,
                            void* dc, void* dz, void* workspace, int accumulate, long long N, int K, float forget_bias,
                            void* stream) {
  if (int e = lstm_ln_args("bsmm_lstm_ln_gates_grad", dtype, gdtype, N, K, stride)) return e;
  if (!c || !z || !g || !b || !mean || !rstd || !dc || !dz || !workspace)
    return fail(BSMM_E_ARG, "bsmm_lstm_ln_gates_grad: null pointer");
  if (N == 0) return 0;
  LnGatesArgs a = {};
  a.c = c; a.z = z; a.g = g; a.b = b; a.mean = (float*)mean; a.rstd = (float*)rstd; a.ec = ec; a.eh = eh;
  a.c_out = dc; a.h_out = dz; a.ws = (float*)workspace; a.accumulate = accumulate != 0;
  a.N = N; a.zs = stride; a.K = K; a.gdt = gdtype; a.forget_bias = forget_bias;
  BSMM_DISPATCH_DTYPE(dtype, T, { return launch_lstm_ln_gates<T>(a, true, (cudaStream_t)stream); });
  return 0;
}

int bsmm_lstm_ln_gates_grad_reduce(int gdtype, const void* workspace, long long N, int K, void* dg, void* db,
                                   void* stream) {
  const char* what = "bsmm_lstm_ln_gates_grad_reduce";
  if (!dense_dtype_ok(gdtype)) return fail(BSMM_E_ARG, "%s: unsupported dtype code %d", what, gdtype);
  if (N < 0 || K <= 0) return fail(BSMM_E_ARG, "%s: bad sizes N %lld, K %d", what, N, K);
  if (K > 0x7fffffff / 4) return fail(BSMM_E_LIMIT, "%s: 4K exceeds 2^31 - 1 (K %d)", what, K);
  if (!workspace || !dg || !db) return fail(BSMM_E_ARG, "%s: null pointer", what);
  if (N == 0) return 0;
  int rpu, parts;
  lng_partition(N, rpu, parts);
  BSMM_DISPATCH_DTYPE(gdtype, G, {
    ln_reduce_partials_kernel<G><<<(unsigned)((4LL * K + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
        (const float*)workspace, parts, 4 * K, dg, db);
  });
  return check_launch("lstm_ln_gates_grad_reduce");
}

int bsmm_sparse_relu(int dtype, const void* x, void* y, long long N, int K, float alpha, void* stream) {
  if (!dense_dtype_ok(dtype)) return fail(BSMM_E_ARG, "bsmm_sparse_relu: unsupported dtype code %d", dtype);
  if (N < 0 || K <= 0) return fail(BSMM_E_ARG, "bsmm_sparse_relu: bad sizes N %lld, K %d", N, K);
  if (!x || !y) return fail(BSMM_E_ARG, "bsmm_sparse_relu: null pointer");
  if (N > LLONG_MAX / K) return fail(BSMM_E_LIMIT, "bsmm_sparse_relu: more than 2^63 elements");
  if (N == 0) return 0;
  SreluArgs a = {};
  a.x = x; a.y = y; a.N = N; a.K = K; a.alpha = alpha;
  const bool vec = aligned16(x) && aligned16(y) && K % (16 / dtype_size(dtype)) == 0;
  BSMM_DISPATCH_DTYPE(dtype, T, { return launch_sparse_relu<T>(a, vec, (cudaStream_t)stream); });
  return 0;
}

int bsmm_relu_mask_grad(int dtype, const void* dy, const void* y, void* dx, long long n, void* stream) {
  if (!dense_dtype_ok(dtype)) return fail(BSMM_E_ARG, "bsmm_relu_mask_grad: unsupported dtype code %d", dtype);
  if (n < 0) return fail(BSMM_E_ARG, "bsmm_relu_mask_grad: bad size %lld", n);
  if (!dy || !y || !dx) return fail(BSMM_E_ARG, "bsmm_relu_mask_grad: null pointer");
  if (n == 0) return 0;
  const bool vec = aligned16(dy) && aligned16(y) && aligned16(dx) && n % (16 / dtype_size(dtype)) == 0;
  BSMM_DISPATCH_DTYPE(dtype, T, { return launch_relu_mask_grad<T>(dy, y, dx, n, vec, (cudaStream_t)stream); });
  return 0;
}

// ---- elementwise math, casts, filters, sums, gates, gathers, column maxima (csrc/elementwise.cuh) -----------------------
static bool all_aligned16(std::initializer_list<const void*> ptrs) {
  for (const void* p : ptrs)
    if (p && !aligned16(p)) return false;
  return true;
}

int bsmm_ew_forward(int dtype, int bdtype, int op, const void* x, const void* y, const void* b, void* z, long long n,
                    long long K, float alpha, void* stream) {
  if (!dense_dtype_ok(dtype)) return fail(BSMM_E_ARG, "bsmm_ew_forward: unsupported dtype code %d", dtype);
  if (op < 0 || op >= EW_NOPS) return fail(BSMM_E_ARG, "bsmm_ew_forward: unknown op code %d", op);
  if (n < 0) return fail(BSMM_E_ARG, "bsmm_ew_forward: bad size %lld", n);
  if (!x || !z || (ew_binary(op) && !y)) return fail(BSMM_E_ARG, "bsmm_ew_forward: null pointer");
  if (ew_bcast(op)) {
    if (!b) return fail(BSMM_E_ARG, "bsmm_ew_forward: null vector");
    if (!dense_dtype_ok(bdtype)) return fail(BSMM_E_ARG, "bsmm_ew_forward: unsupported vector dtype code %d", bdtype);
    if (K <= 0 || n % K) return fail(BSMM_E_ARG, "bsmm_ew_forward: n %lld is not a multiple of K %lld", n, K);
  }
  if (n == 0) return 0;
  EwArgs a = {};
  a.x = x; a.y = y; a.b = b; a.z = z; a.n = n; a.K = K; a.bdt = bdtype; a.alpha = alpha;
  const bool vec = all_aligned16({x, ew_binary(op) ? y : nullptr, z}) && (!ew_bcast(op) || K % (16 / dtype_size(dtype)) == 0);
  BSMM_DISPATCH_DTYPE(dtype, T, { return launch_ew<T>(a, op, false, vec, (cudaStream_t)stream); });
  return 0;
}

int bsmm_ew_backward(int dtype, int op, const void* dz, const void* x, const void* y, void* dx, void* dy, long long n,
                     float alpha, void* stream) {
  if (!dense_dtype_ok(dtype)) return fail(BSMM_E_ARG, "bsmm_ew_backward: unsupported dtype code %d", dtype);
  if (op < 0 || op >= EW_NOPS || op == EW_ADD || op == EW_SUB || op == EW_NEG || ew_bcast(op))
    return fail(BSMM_E_ARG, "bsmm_ew_backward: op code %d has no backward kernel", op);
  if (n < 0) return fail(BSMM_E_ARG, "bsmm_ew_backward: bad size %lld", n);
  if (!dz || !x || !dx || (ew_binary(op) && (!y || !dy))) return fail(BSMM_E_ARG, "bsmm_ew_backward: null pointer");
  if (n == 0) return 0;
  EwArgs a = {};
  a.dz = dz; a.x = x; a.y = y; a.z = dx; a.dy = dy; a.n = n; a.alpha = alpha;
  const bool vec = all_aligned16({dz, x, dx, ew_binary(op) ? y : nullptr, ew_binary(op) ? dy : nullptr});
  BSMM_DISPATCH_DTYPE(dtype, T, { return launch_ew<T>(a, op, true, vec, (cudaStream_t)stream); });
  return 0;
}

int bsmm_gain_mul_grad(int dtype, int gdtype, const void* dz, const void* x, const void* g, void* dx, void* dg,
                       void* workspace, long long N, int K, void* stream) {
  if (!dense_dtype_ok(dtype) || !dense_dtype_ok(gdtype))
    return fail(BSMM_E_ARG, "bsmm_gain_mul_grad: unsupported dtype codes %d, %d", dtype, gdtype);
  if (N < 0 || K <= 0) return fail(BSMM_E_ARG, "bsmm_gain_mul_grad: bad sizes N %lld, K %d", N, K);
  if (!dz || !x || !g || !dx || !dg || !workspace) return fail(BSMM_E_ARG, "bsmm_gain_mul_grad: null pointer");
  if (N > LLONG_MAX / K) return fail(BSMM_E_LIMIT, "bsmm_gain_mul_grad: more than 2^63 elements");
  if (N == 0) return 0;
  BrArgs a = {};
  a.x = x; a.b = g; a.y = dx; a.part = (float*)workspace; a.N = N; a.K = K; a.bdt = gdtype;
  const bool vec = all_aligned16({dz, x, dx}) && K % (16 / dtype_size(dtype)) == 0;
  BSMM_DISPATCH_DTYPE(dtype, T, { return launch_gain_mul_grad<T>(a, dz, dg, vec, (cudaStream_t)stream); });
  return 0;
}

int bsmm_float_cast(int xdtype, int ydtype, const void* x, void* y, long long n, void* stream) {
  if (!dense_dtype_ok(xdtype) || !dense_dtype_ok(ydtype))
    return fail(BSMM_E_ARG, "bsmm_float_cast: unsupported dtype codes %d, %d", xdtype, ydtype);
  if (n < 0) return fail(BSMM_E_ARG, "bsmm_float_cast: bad size %lld", n);
  if (!x || !y) return fail(BSMM_E_ARG, "bsmm_float_cast: null pointer");
  if (n == 0) return 0;
  return launch_float_cast(xdtype, ydtype, x, y, n, all_aligned16({x, y}), (cudaStream_t)stream);
}

int bsmm_filter_tensor(int dtype, const void* x, void* y, long long n, float scale, const float* scale_ptr,
                       float saturate, int zero_infs, int zero_nans, void* stream) {
  if (!dense_dtype_ok(dtype)) return fail(BSMM_E_ARG, "bsmm_filter_tensor: unsupported dtype code %d", dtype);
  if (n < 0) return fail(BSMM_E_ARG, "bsmm_filter_tensor: bad size %lld", n);
  if (!x || !y) return fail(BSMM_E_ARG, "bsmm_filter_tensor: null pointer");
  if (n == 0) return 0;
  FilterArgs a = {};
  a.x = x; a.y = y; a.scale_ptr = scale_ptr; a.n = n; a.scale = scale; a.saturate = saturate;
  a.zero_infs = zero_infs != 0; a.zero_nans = zero_nans != 0;
  BSMM_DISPATCH_DTYPE(dtype, T, { return launch_filter<T>(a, all_aligned16({x, y}), (cudaStream_t)stream); });
  return 0;
}

int bsmm_add_n(int dtype, const void* const* xs, int count, void* y, long long n, void* stream) {
  if (!dense_dtype_ok(dtype)) return fail(BSMM_E_ARG, "bsmm_add_n: unsupported dtype code %d", dtype);
  if (count < 1 || count > ADDN_MAX) return fail(BSMM_E_ARG, "bsmm_add_n: count must be in [1, %d], got %d", ADDN_MAX, count);
  if (n < 0) return fail(BSMM_E_ARG, "bsmm_add_n: bad size %lld", n);
  if (!xs || !y) return fail(BSMM_E_ARG, "bsmm_add_n: null pointer");
  AddNArgs a = {};
  bool vec = aligned16(y);
  for (int i = 0; i < count; ++i) {
    if (!xs[i]) return fail(BSMM_E_ARG, "bsmm_add_n: null input %d", i);
    a.x[i] = xs[i];
    vec = vec && aligned16(xs[i]);
  }
  if (n == 0) return 0;
  a.y = y; a.n = n; a.count = count;
  BSMM_DISPATCH_DTYPE(dtype, T, { return launch_add_n<T>(a, vec, (cudaStream_t)stream); });
  return 0;
}

static int gate_args(const char* what, int dtype, long long n, float limit_a, float limit_b) {
  if (!dense_dtype_ok(dtype)) return fail(BSMM_E_ARG, "%s: unsupported dtype code %d", what, dtype);
  if (n < 0) return fail(BSMM_E_ARG, "%s: bad size %lld", what, n);
  if (!(limit_a < limit_b)) return fail(BSMM_E_ARG, "%s: limit_a %g must be below limit_b %g", what, limit_a, limit_b);
  return 0;
}

int bsmm_concrete_gate(int dtype, const void* loga, void* gate, float* concrete, long long n, float rcp_temp,
                       float limit_a, float limit_b, float epsilon, long long* state, void* stream) {
  if (int e = gate_args("bsmm_concrete_gate", dtype, n, limit_a, limit_b)) return e;
  if (!loga || !gate || !concrete || !state) return fail(BSMM_E_ARG, "bsmm_concrete_gate: null pointer");
  if (!(epsilon >= 0.f && epsilon < 0.5f)) return fail(BSMM_E_ARG, "bsmm_concrete_gate: epsilon must be in [0, 0.5)");
  if (n == 0) return 0;
  GateArgs a = {};
  a.loga = loga; a.gate = gate; a.concrete = concrete; a.state = state; a.n = n; a.rcp_temp = rcp_temp;
  a.limit_a = limit_a; a.limit_b = limit_b; a.epsilon = epsilon;
  BSMM_DISPATCH_DTYPE(dtype, T, { return launch_concrete_gate<T>(a, 0, (cudaStream_t)stream); });
  return 0;
}

int bsmm_concrete_gate_grad(int dtype, const void* dgate, const float* concrete, void* dloga, long long n,
                            float rcp_temp, float limit_a, float limit_b, void* stream) {
  if (int e = gate_args("bsmm_concrete_gate_grad", dtype, n, limit_a, limit_b)) return e;
  if (!dgate || !concrete || !dloga) return fail(BSMM_E_ARG, "bsmm_concrete_gate_grad: null pointer");
  if (n == 0) return 0;
  GateArgs a = {};
  a.loga = dgate; a.gate = dloga; a.concrete = (float*)concrete; a.n = n; a.rcp_temp = rcp_temp;
  a.limit_a = limit_a; a.limit_b = limit_b;
  BSMM_DISPATCH_DTYPE(dtype, T, { return launch_concrete_gate<T>(a, 1, (cudaStream_t)stream); });
  return 0;
}

int bsmm_concrete_gate_infer(int dtype, const void* loga, void* gate, long long n, float limit_a, float limit_b,
                             void* stream) {
  if (int e = gate_args("bsmm_concrete_gate_infer", dtype, n, limit_a, limit_b)) return e;
  if (!loga || !gate) return fail(BSMM_E_ARG, "bsmm_concrete_gate_infer: null pointer");
  if (n == 0) return 0;
  GateArgs a = {};
  a.loga = loga; a.gate = gate; a.n = n; a.limit_a = limit_a; a.limit_b = limit_b;
  BSMM_DISPATCH_DTYPE(dtype, T, { return launch_concrete_gate<T>(a, 2, (cudaStream_t)stream); });
  return 0;
}

static int dims3(const char* what, long long d0, long long d1, long long d2) {
  if (d0 < 0 || d1 < 0 || d2 < 0) return fail(BSMM_E_ARG, "%s: bad dims %lld, %lld, %lld", what, d0, d1, d2);
  if (d0 && d1 && d2 && (d1 > LLONG_MAX / d2 || d0 > LLONG_MAX / (d1 * d2)))
    return fail(BSMM_E_LIMIT, "%s: more than 2^63 elements", what);
  return 0;
}

int bsmm_fancy_gather(int esize, const void* x, const int32_t* idx, void* y, long long d0, long long d1, long long d2,
                      void* stream) {
  if (esize != 2 && esize != 4) return fail(BSMM_E_ARG, "bsmm_fancy_gather: element size must be 2 or 4, got %d", esize);
  if (int e = dims3("bsmm_fancy_gather", d0, d1, d2)) return e;
  if (!x || !idx || !y) return fail(BSMM_E_ARG, "bsmm_fancy_gather: null pointer");
  if (d0 * d2 == 0) return 0;
  return launch_fancy_gather(esize, false, x, idx, y, d0, d1, d2, (cudaStream_t)stream);
}

int bsmm_fancy_gather_grad(int esize, const void* dy, const int32_t* idx, void* dx, long long d0, long long d1,
                           long long d2, void* stream) {
  if (esize != 2 && esize != 4) return fail(BSMM_E_ARG, "bsmm_fancy_gather_grad: element size must be 2 or 4, got %d", esize);
  if (int e = dims3("bsmm_fancy_gather_grad", d0, d1, d2)) return e;
  if (!dy || !idx || !dx) return fail(BSMM_E_ARG, "bsmm_fancy_gather_grad: null pointer");
  if (d0 * d1 * d2 == 0) return 0;
  return launch_fancy_gather(esize, true, dy, idx, dx, d0, d1, d2, (cudaStream_t)stream);
}

static int rmax_args(const char* what, int dtype, int idx_type, long long d0, long long d1, long long d2) {
  if (!dense_dtype_ok(dtype)) return fail(BSMM_E_ARG, "%s: unsupported dtype code %d", what, dtype);
  if (idx_type != BSMM_LABEL_U8 && idx_type != BSMM_LABEL_U16 && idx_type != BSMM_LABEL_I32)
    return fail(BSMM_E_ARG, "%s: index type %d is not U8, U16 or I32", what, idx_type);
  if (int e = dims3(what, d0, d1, d2)) return e;
  if (d1 < 1) return fail(BSMM_E_ARG, "%s: the reduced dim must have at least one entry", what);
  const long long cap = idx_type == BSMM_LABEL_U8 ? 256 : idx_type == BSMM_LABEL_U16 ? 65536 : 2147483648LL;
  if (d1 > cap) return fail(BSMM_E_ARG, "%s: %lld entries do not fit index type %d", what, d1, idx_type);
  return 0;
}

int bsmm_reduce_max(int dtype, int idx_type, const void* x, void* y, void* argmax, long long d0, long long d1,
                    long long d2, void* stream) {
  if (int e = rmax_args("bsmm_reduce_max", dtype, idx_type, d0, d1, d2)) return e;
  if (!x || !y || !argmax) return fail(BSMM_E_ARG, "bsmm_reduce_max: null pointer");
  if (d0 * d2 == 0) return 0;
  BSMM_DISPATCH_DTYPE(dtype, T, {
    return launch_reduce_max<T>(idx_type, false, x, argmax, nullptr, y, d0, d1, d2, (cudaStream_t)stream);
  });
  return 0;
}

int bsmm_reduce_max_grad(int dtype, int idx_type, const void* dy, const void* argmax, void* dx, long long d0,
                         long long d1, long long d2, void* stream) {
  if (int e = rmax_args("bsmm_reduce_max_grad", dtype, idx_type, d0, d1, d2)) return e;
  if (!dy || !argmax || !dx) return fail(BSMM_E_ARG, "bsmm_reduce_max_grad: null pointer");
  if (d0 * d2 == 0) return 0;
  BSMM_DISPATCH_DTYPE(dtype, T, {
    return launch_reduce_max<T>(idx_type, true, dy, (void*)argmax, dx, nullptr, d0, d1, d2, (cudaStream_t)stream);
  });
  return 0;
}

// ---- embedding (csrc/embed.cuh) --------------------------------------------------------------------------------------------
static int emb_args(const char* what, int dtype, int idx_type, long long n, int C, int K) {
  if (!dense_dtype_ok(dtype)) return fail(BSMM_E_ARG, "%s: unsupported dtype code %d", what, dtype);
  if (idx_type < BSMM_LABEL_U8 || idx_type > BSMM_LABEL_I64) return fail(BSMM_E_ARG, "%s: unsupported index type %d", what, idx_type);
  if (n < 0 || C < 0 || K <= 0) return fail(BSMM_E_ARG, "%s: bad sizes n %lld, C %d, K %d", what, n, C, K);
  return 0;
}

int bsmm_embedding_lookup(int dtype, int idx_type, const void* emb, const void* idx, void* y, long long n, int C, int K,
                          void* stream) {
  if (int e = emb_args("bsmm_embedding_lookup", dtype, idx_type, n, C, K)) return e;
  if (!idx || !y || (C > 0 && !emb)) return fail(BSMM_E_ARG, "bsmm_embedding_lookup: null pointer");
  if (n == 0) return 0;
  const int es = dtype_size(dtype);
  if (aligned16(emb) && aligned16(y) && (K * es) % 16 == 0)
    return launch_embedding_lookup<uint4>(emb, idx, idx_type, y, n, C, K * es / 16, (cudaStream_t)stream);
  if (es == 4) return launch_embedding_lookup<uint32_t>(emb, idx, idx_type, y, n, C, K, (cudaStream_t)stream);
  return launch_embedding_lookup<uint16_t>(emb, idx, idx_type, y, n, C, K, (cudaStream_t)stream);
}

size_t bsmm_embedding_grad_workspace_bytes(long long n, int C, int K) {
  if (n <= 0 || n > 0x7fffffffLL || C <= 0 || C == INT_MAX || K <= 0) return 0;
  return emb_workspace_bytes(n, C, K);
}

int bsmm_embedding_grad(int dtype, int idx_type, const void* dy, const void* idx, void* dw, void* workspace, long long n,
                        int C, int K, void* stream) {
  if (int e = emb_args("bsmm_embedding_grad", dtype, idx_type, n, C, K)) return e;
  if (!idx || !dy || !dw || (n > 0 && !workspace)) return fail(BSMM_E_ARG, "bsmm_embedding_grad: null pointer");
  if (n > 0x7fffffffLL) return fail(BSMM_E_LIMIT, "bsmm_embedding_grad: more than 2^31 - 1 indices");
  if (C == INT_MAX) return fail(BSMM_E_LIMIT, "bsmm_embedding_grad: C must be below 2^31 - 1");
  if (C == 0 || n == 0) return 0;
  const bool vec = aligned16(dy) && aligned16(dw) && K % (16 / dtype_size(dtype)) == 0;
  BSMM_DISPATCH_DTYPE(dtype, T, {
    return launch_embedding_grad<T>(dy, idx, idx_type, dw, workspace, n, C, K, vec, (cudaStream_t)stream);
  });
  return 0;
}

// ---------------------------------------------------------------------------------------
struct Timer { cudaEvent_t start, stop; };

int bsmm_timer_create(void** timer) {
  if (!timer) return fail(BSMM_E_ARG, "null timer");
  Timer* t = new Timer;
  if (cudaEventCreate(&t->start) != cudaSuccess || cudaEventCreate(&t->stop) != cudaSuccess) {
    delete t;
    return fail(BSMM_E_NODEV, "cudaEventCreate failed");
  }
  *timer = t;
  return 0;
}
int bsmm_timer_begin(void* timer, void* stream) {
  if (!timer) return fail(BSMM_E_ARG, "null timer");
  return (int)cudaEventRecord(((Timer*)timer)->start, (cudaStream_t)stream);
}
int bsmm_timer_end(void* timer, void* stream, float* ms_out) {
  if (!timer || !ms_out) return fail(BSMM_E_ARG, "null timer");
  Timer* t = (Timer*)timer;
  cudaError_t e = cudaEventRecord(t->stop, (cudaStream_t)stream);
  if (e == cudaSuccess) e = cudaEventSynchronize(t->stop);
  if (e == cudaSuccess) e = cudaEventElapsedTime(ms_out, t->start, t->stop);
  if (e != cudaSuccess) return fail((int)e, "timer: %s", cudaGetErrorString(e));
  return 0;
}
int bsmm_timer_destroy(void* timer) {
  if (!timer) return 0;
  Timer* t = (Timer*)timer;
  cudaEventDestroy(t->start); cudaEventDestroy(t->stop);
  delete t;
  return 0;
}


// ---- weight utilities (csrc/wutil.cuh) ---------------------------------------------------------------------------
static int check_blocks(const char* what, int bsize, int blocks, const void* p) {
  if (!p || blocks <= 0) return fail(BSMM_E_ARG, "%s: bad arguments", what);
  return check_bsize_axis(bsize, 0);
}

int bsmm_block_norm(int dtype, int bsize, int blocks, const void* w, float* norm, int norm_type, void* stream) {
  if (int e = check_blocks("bsmm_block_norm", bsize, blocks, w)) return e;
  if (!norm) return fail(BSMM_E_ARG, "bsmm_block_norm: null output");
  const int wpb = 4;
  BSMM_DISPATCH_DTYPE(dtype, T, {
    block_norm_kernel<T><<<(blocks + wpb - 1) / wpb, wpb * 32, 0, (cudaStream_t)stream>>>((const T*)w, norm, blocks, bsize * bsize, norm_type != 0);
  });
  return check_launch("block_norm");
}

int bsmm_l2_decay(int dtype, int bsize, int blocks, void* w, const float* gate, float rate, float epsilon, void* stream) {
  if (int e = check_blocks("bsmm_l2_decay", bsize, blocks, w)) return e;
  const int wpb = 4;
  BSMM_DISPATCH_DTYPE(dtype, T, {
    l2_decay_kernel<T><<<(blocks + wpb - 1) / wpb, wpb * 32, 0, (cudaStream_t)stream>>>((T*)w, gate, blocks, bsize * bsize, rate, epsilon);
  });
  return check_launch("l2_decay");
}

int bsmm_threshold_prune(int dtype, int bsize, int blocks, const void* w, float* gate, float threshold, int norm_type, void* stream) {
  if (int e = check_blocks("bsmm_threshold_prune", bsize, blocks, w)) return e;
  if (!gate) return fail(BSMM_E_ARG, "bsmm_threshold_prune: null gate");
  const int wpb = 4;
  BSMM_DISPATCH_DTYPE(dtype, T, {
    threshold_prune_kernel<T><<<(blocks + wpb - 1) / wpb, wpb * 32, 0, (cudaStream_t)stream>>>((const T*)w, gate, blocks, bsize * bsize, threshold, norm_type != 0);
  });
  return check_launch("threshold_prune");
}

int bsmm_prune_topk(float* gate, const int32_t* idx, int blocks, int keep, void* stream) {
  if (!gate || !idx || blocks <= 0 || keep < 0) return fail(BSMM_E_ARG, "bsmm_prune_topk: bad arguments");
  prune_topk_kernel<<<(blocks + 255) / 256, 256, 0, (cudaStream_t)stream>>>(gate, idx, blocks, keep);
  return check_launch("prune_topk");
}

int bsmm_identity_init(int dtype, int bsize, int blocks, const int32_t* updat_lut, int n_c_blocks, int n_k_blocks, void* w, float scale, void* stream) {
  if (int e = check_blocks("bsmm_identity_init", bsize, blocks, w)) return e;
  if (!updat_lut || n_c_blocks <= 0 || n_k_blocks <= 0) return fail(BSMM_E_ARG, "bsmm_identity_init: bad arguments");
  BSMM_DISPATCH_DTYPE(dtype, T, {
    identity_init_kernel<T><<<blocks, 128, 0, (cudaStream_t)stream>>>((T*)w, updat_lut, blocks, bsize, n_c_blocks, n_k_blocks, scale);
  });
  return check_launch("identity_init");
}

int bsmm_l2_normalize(int dtype, int y_dtype, int bsize, const int32_t* lut, int n_out, const void* w, const float* gain, void* y,
                      float* sum_sqr, float epsilon, void* stream) {
  if (int e = check_bsize_axis(bsize, 0)) return e;
  if (!lut || !w || !y || !sum_sqr || n_out <= 0) return fail(BSMM_E_ARG, "bsmm_l2_normalize: bad arguments");
  if (y_dtype != dtype && y_dtype != BSMM_F32) return fail(BSMM_E_DTYPE, "bsmm_l2_normalize: output dtype must be fp32 or the input dtype");
  cudaStream_t s = (cudaStream_t)stream;
  BSMM_DISPATCH_DTYPE(dtype, T, {
    if (y_dtype == BSMM_F32) l2_normalize_kernel<T, float><<<n_out, L2N_THREADS, 0, s>>>((const T*)w, gain, (float*)y, sum_sqr, lut, bsize, epsilon);
    else                     l2_normalize_kernel<T, T><<<n_out, L2N_THREADS, 0, s>>>((const T*)w, gain, (T*)y, sum_sqr, lut, bsize, epsilon);
  });
  return check_launch("l2_normalize");
}

int bsmm_l2_normalize_grad(int dtype, int y_dtype, int bsize, const int32_t* lut, int n_out, const void* dy, const void* w, const float* gain,
                           const float* sum_sqr, void* dx, float* dg, float epsilon, void* stream) {
  if (int e = check_bsize_axis(bsize, 0)) return e;
  if (!lut || !dy || !w || !sum_sqr || !dx || n_out <= 0) return fail(BSMM_E_ARG, "bsmm_l2_normalize_grad: bad arguments");
  if (y_dtype != dtype && y_dtype != BSMM_F32) return fail(BSMM_E_DTYPE, "bsmm_l2_normalize_grad: dy dtype must be fp32 or the weight dtype");
  cudaStream_t s = (cudaStream_t)stream;
  BSMM_DISPATCH_DTYPE(dtype, T, {
    if (y_dtype == BSMM_F32) l2_normalize_grad_kernel<T, float><<<n_out, L2N_THREADS, 0, s>>>((const float*)dy, (const T*)w, gain, sum_sqr, (T*)dx, dg, lut, bsize, epsilon);
    else                     l2_normalize_grad_kernel<T, T><<<n_out, L2N_THREADS, 0, s>>>((const T*)dy, (const T*)w, gain, sum_sqr, (T*)dx, dg, lut, bsize, epsilon);
  });
  return check_launch("l2_normalize_grad");
}

size_t bsmm_reduced_dw_workspace_bytes(int n_c_blocks, int n_k_blocks) { return (size_t)8 * n_c_blocks * n_k_blocks * sizeof(float); }

int bsmm_reduced_dw(int dtype, int axis, int bsize, const void* const* xs, const void* const* dys, int pcount,
                    int n_c_blocks, int n_k_blocks, int N, float scale, int norm_type, float* dw, int accumulate,
                    void* x_red, void* y_red, void* workspace, void* stream) {
  if (int e = check_bsize_axis(bsize, axis)) return e;
  if (!xs || !dys || !dw || !x_red || !y_red || !workspace) return fail(BSMM_E_ARG, "bsmm_reduced_dw: null pointer");
  if (pcount < 1 || pcount > BSMM_MAX_PAIRS || n_c_blocks <= 0 || n_k_blocks <= 0 || N <= 0) return fail(BSMM_E_ARG, "bsmm_reduced_dw: bad sizes");
  if (dtype != BSMM_F16 && dtype != BSMM_BF16) return fail(BSMM_E_DTYPE, "bsmm_reduced_dw: 16-bit activations only (reference: half)");
  cudaStream_t s = (cudaStream_t)stream;
  const int total = n_c_blocks * n_k_blocks;
  if (scale == 0.0f) {          // a zero scale computes nothing (reference op.cc:754-766; its hGemmNT / hGemmTN return early)
    const size_t per_block = (size_t)pcount * N * 2;        // 16-bit x_red / y_red elements of one feature block
    cudaError_t e = cudaMemsetAsync(x_red, 0, per_block * n_c_blocks, s);
    if (e == cudaSuccess) e = cudaMemsetAsync(y_red, 0, per_block * n_k_blocks, s);
    if (e == cudaSuccess && !accumulate) e = cudaMemsetAsync(dw, 0, (size_t)total * sizeof(float), s);
    if (e != cudaSuccess) return fail((int)e, "reduced_dw: %s", cudaGetErrorString(e));
    return check_launch("reduced_dw");
  }
  const int l2 = norm_type != 0;
  const int splits = 8;
  BSMM_DISPATCH_DTYPE(dtype, T, {
    for (int p = 0; p < pcount; ++p) {
      if (!xs[p] || !dys[p]) return fail(BSMM_E_ARG, "bsmm_reduced_dw: null pointer in pair %d", p);
      const long long tx = (long long)n_c_blocks * N, ty = (long long)n_k_blocks * N;
      feature_reduce_kernel<T><<<(unsigned)((tx + 255) / 256), 256, 0, s>>>((const T*)xs[p], (T*)x_red, axis, bsize, n_c_blocks, N, p, pcount, l2);
      feature_reduce_kernel<T><<<(unsigned)((ty + 255) / 256), 256, 0, s>>>((const T*)dys[p], (T*)y_red, axis, bsize, n_k_blocks, N, p, pcount, l2);
    }
    const long long R = (long long)pcount * N;
    dim3 grid((n_c_blocks + 15) / 16, (n_k_blocks + 15) / 16, splits);
    if (axis == 1)     // (pair, n, block): row r = pair*N + n, block contiguous
      reduced_gemm_partial_kernel<T><<<grid, 256, 0, s>>>((const T*)x_red, (const T*)y_red, (float*)workspace, n_c_blocks, n_k_blocks, R,
                                                          n_c_blocks, 1, n_k_blocks, 1, splits);
    else               // (block, pair, n): row r = pair*N + n contiguous, block stride R
      reduced_gemm_partial_kernel<T><<<grid, 256, 0, s>>>((const T*)x_red, (const T*)y_red, (float*)workspace, n_c_blocks, n_k_blocks, R,
                                                          1, R, 1, R, splits);
  });
  reduced_gemm_finish_kernel<<<(total + 255) / 256, 256, 0, s>>>((const float*)workspace, dw, total, splits, scale, accumulate);
  return check_launch("reduced_dw");
}

int bsmm_gather_rows(int dtype, const void* x, const void* y, const int32_t* idx, void* out, int rows, long long N, int op, void* stream) {
  if (!x || !idx || !out || rows <= 0 || N <= 0 || op < 0 || op > 2 || (op != 0 && !y)) return fail(BSMM_E_ARG, "bsmm_gather_rows: bad arguments");
  const unsigned gy = (unsigned)((N + 255) / 256 > 64 ? 64 : (N + 255) / 256);
  BSMM_DISPATCH_DTYPE(dtype, T, {
    gather_rows_kernel<T><<<dim3(rows, gy), 256, 0, (cudaStream_t)stream>>>((const T*)x, (const T*)y, idx, (T*)out, rows, N, op);
  });
  return check_launch("gather_rows");
}

int bsmm_pad_blocks(int dtype, int bsize, int blocks_big, const int32_t* sub_map, const void* w_small, const float* gate, void* w_big, void* stream) {
  if (!sub_map || !w_small || !w_big || blocks_big <= 0 || (bsize != 8 && bsize != 16 && bsize != 32)) return fail(BSMM_E_ARG, "bsmm_pad_blocks: bad arguments");
  BSMM_DISPATCH_DTYPE(dtype, T, {
    pad_blocks_kernel<T><<<blocks_big, 128, 0, (cudaStream_t)stream>>>((const T*)w_small, sub_map, gate, (T*)w_big, blocks_big, bsize);
  });
  return check_launch("pad_blocks");
}

int bsmm_unpad_blocks(int in_dtype, int out_dtype, int bsize, int blocks_small, const int32_t* inv_map, const void* dw_big, const float* gate,
                      void* dw_small, int accumulate, void* stream) {
  if (!inv_map || !dw_big || !dw_small || blocks_small <= 0 || (bsize != 8 && bsize != 16 && bsize != 32)) return fail(BSMM_E_ARG, "bsmm_unpad_blocks: bad arguments");
  cudaStream_t s = (cudaStream_t)stream;
  BSMM_DISPATCH_DTYPE(in_dtype, TI, {
    BSMM_DISPATCH_DTYPE(out_dtype, TO, {
      unpad_blocks_kernel<TI, TO><<<blocks_small, 64, 0, s>>>((const TI*)dw_big, inv_map, gate, (TO*)dw_small, blocks_small, bsize, accumulate);
    });
  });
  return check_launch("unpad_blocks");
}

// ---- optimizer (csrc/optimize.cuh) ----------------------------------------------------------------------------------------
// Validates tensor i of a multi-tensor call: size >= 0, a known dtype, non-null pointers where the tensor has elements, and
// for a gated tensor bs in {8, 16, 32, 64}, a gate and a size that is a multiple of bs*bs.
static int mt_check(const char* what, int i, long long size, int dtype, const void* const* ptrs, int nptr, const float* gate,
                    int bsize) {
  if (size < 0) return fail(BSMM_E_ARG, "%s: tensor %d has negative size %lld", what, i, size);
  if (!dense_dtype_ok(dtype)) return fail(BSMM_E_ARG, "%s: tensor %d has unsupported dtype code %d", what, i, dtype);
  if (bsize != 0 && bsize != 8 && bsize != 16 && bsize != 32 && bsize != 64)
    return fail(BSMM_E_ARG, "%s: tensor %d has block size %d (0, 8, 16, 32 or 64)", what, i, bsize);
  if (bsize && size % ((long long)bsize * bsize))
    return fail(BSMM_E_ARG, "%s: tensor %d of %lld elements is not made of %d x %d blocks", what, i, size, bsize, bsize);
  if (mt_chunks(size) > 0x7fffffffLL) return fail(BSMM_E_LIMIT, "%s: tensor %d of %lld elements exceeds the grid", what, i, size);
  if (size == 0) return 0;
  for (int j = 0; j < nptr; ++j)
    if (!ptrs[j]) return fail(BSMM_E_ARG, "%s: tensor %d has a null pointer", what, i);
  if (bsize && !gate) return fail(BSMM_E_ARG, "%s: tensor %d is gated without a gate", what, i);
  return 0;
}

static uint8_t mt_bshift(int bsize) { return bsize ? (uint8_t)(2 * (31 - __builtin_clz((unsigned)bsize))) : 0; }

int bsmm_adam(int n, const void* const* grads, const int* grad_dtypes, float* const* params, void* const* means,
              void* const* vars, const int* moment_codes, const long long* sizes, const float* const* gates,
              const int* bsizes, const float* norm_scale, float lr, float decay_mean, float decay_var, float epsilon,
              float grad_scale, float clip_sigma, float saturate, int zero_infs, int zero_nans, void* stream) {
  if (n < 0) return fail(BSMM_E_ARG, "bsmm_adam: n = %d", n);
  if (n && (!grads || !grad_dtypes || !params || !means || !vars || !moment_codes || !sizes))
    return fail(BSMM_E_ARG, "bsmm_adam: null array");
  for (int i = 0; i < n; ++i) {
    const void* ptrs[4] = {grads[i], params[i], means[i], vars[i]};
    const int bs = bsizes ? bsizes[i] : 0;
    if (moment_codes[i] != 0 && moment_codes[i] != 1)
      return fail(BSMM_E_ARG, "bsmm_adam: tensor %d has moment code %d (0 or 1)", i, moment_codes[i]);
    if (int e = mt_check("bsmm_adam", i, sizes[i], grad_dtypes[i], ptrs, 4, bs && gates ? gates[i] : nullptr, bs)) return e;
  }
  AdamConsts k = {norm_scale, lr, decay_mean, decay_var, epsilon, grad_scale, clip_sigma, saturate, zero_infs, zero_nans};
  return mt_for_launches(n, sizes,
      [&](int i, MtTensor& t) {
        t.a = grads[i]; t.b = params[i]; t.c = means[i]; t.d = vars[i];
        const int bs = bsizes ? bsizes[i] : 0;
        t.gate = bs ? gates[i] : nullptr; t.bshift = mt_bshift(bs);
        t.dtype = (uint8_t)grad_dtypes[i]; t.codes = (uint8_t)moment_codes[i];
        t.vec = aligned16(t.a) && aligned16(t.b) && aligned16(t.c) && aligned16(t.d);
      },
      [&](const MtTable& tab, int chunks, long long) {
        mt_adam<<<chunks, MT_THREADS, 0, (cudaStream_t)stream>>>(tab, k);
        return check_launch("mt_adam");
      });
}

size_t bsmm_global_norm_workspace_bytes(int n, const long long* sizes) {
  if (n < 0 || (n && !sizes)) return 0;
  long long chunks = 0;
  for (int i = 0; i < n; ++i) {
    if (sizes[i] < 0) return 0;
    chunks += mt_chunks(sizes[i]);
  }
  return (size_t)chunks * sizeof(float);
}

int bsmm_global_norm(int n, const void* const* xs, const int* dtypes, const long long* sizes, float grad_scale,
                     float clip_norm, float saturate, int zero_infs, int zero_nans, float* norm, float* scale,
                     void* workspace, void* stream) {
  if (n < 0) return fail(BSMM_E_ARG, "bsmm_global_norm: n = %d", n);
  if (n && (!xs || !dtypes || !sizes)) return fail(BSMM_E_ARG, "bsmm_global_norm: null array");
  if (!norm || !scale) return fail(BSMM_E_ARG, "bsmm_global_norm: null output");
  long long total = 0;
  for (int i = 0; i < n; ++i) {
    if (int e = mt_check("bsmm_global_norm", i, sizes[i], dtypes[i], &xs[i], 1, nullptr, 0)) return e;
    total += mt_chunks(sizes[i]);
  }
  if (total == 0) return 0;                          // nothing launched: norm and scale are left to the caller (0 and 1)
  if (total > 0x7fffffffLL) return fail(BSMM_E_LIMIT, "bsmm_global_norm: %lld chunks exceed the grid", total);
  if (!workspace) return fail(BSMM_E_ARG, "bsmm_global_norm: null workspace");
  float* partial = static_cast<float*>(workspace);
  const NormConsts k = {grad_scale, saturate, zero_infs, zero_nans};
  if (int e = mt_for_launches(n, sizes,
          [&](int i, MtTensor& t) { t.a = xs[i]; t.dtype = (uint8_t)dtypes[i]; t.vec = aligned16(t.a); },
          [&](const MtTable& tab, int chunks, long long base) {
            mt_sumsq<<<chunks, MT_THREADS, 0, (cudaStream_t)stream>>>(tab, k, partial + base);
            return check_launch("mt_sumsq");
          }))
    return e;
  mt_norm_finish<<<1, MT_NORM_THREADS, 0, (cudaStream_t)stream>>>(partial, (int)total, clip_norm, norm, scale);
  return check_launch("mt_norm_finish");
}

int bsmm_ema(int n, void* const* emas, int ema_dtype, const float* const* params, const long long* sizes,
             const float* const* gates, const int* bsizes, float decay, void* stream) {
  if (n < 0) return fail(BSMM_E_ARG, "bsmm_ema: n = %d", n);
  if (ema_dtype != BSMM_F32 && ema_dtype != BSMM_F16) return fail(BSMM_E_ARG, "bsmm_ema: ema dtype %d (F32 or F16)", ema_dtype);
  if (n && (!emas || !params || !sizes)) return fail(BSMM_E_ARG, "bsmm_ema: null array");
  for (int i = 0; i < n; ++i) {
    const void* ptrs[2] = {emas[i], params[i]};
    const int bs = bsizes ? bsizes[i] : 0;
    if (int e = mt_check("bsmm_ema", i, sizes[i], ema_dtype, ptrs, 2, bs && gates ? gates[i] : nullptr, bs)) return e;
  }
  return mt_for_launches(n, sizes,
      [&](int i, MtTensor& t) {
        t.a = params[i]; t.b = emas[i];
        const int bs = bsizes ? bsizes[i] : 0;
        t.gate = bs ? gates[i] : nullptr; t.bshift = mt_bshift(bs);
        t.dtype = (uint8_t)ema_dtype; t.vec = aligned16(t.a) && aligned16(t.b);
      },
      [&](const MtTable& tab, int chunks, long long) {
        if (ema_dtype == BSMM_F32) {
          mt_ema<float><<<chunks, MT_THREADS, 0, (cudaStream_t)stream>>>(tab, decay);
          return check_launch("mt_ema");
        }
        mt_ema<__half><<<chunks, MT_THREADS, 0, (cudaStream_t)stream>>>(tab, decay);
        return check_launch("mt_ema_f16");
      });
}

size_t bsmm_adafactor_workspace_bytes(int n, const long long* rows, const long long* cols) {
  if (n < 0 || (n && (!rows || !cols))) return 0;
  long long floats = 0;
  for (int i = 0; i < n; ++i) {
    if (rows[i] < 0 || cols[i] < 0) return 0;
    floats += af_ws_floats(rows[i], cols[i]);
  }
  return (size_t)floats * sizeof(float);
}

int bsmm_adafactor(int n, const void* const* grads, const int* grad_dtypes, float* const* params, float* const* cvs,
                   float* const* rvs, const long long* rows, const long long* cols, const float* norm_scale, float lr,
                   float decay, float epsilon, float grad_scale, float clip_thresh, float saturate, int zero_infs,
                   int zero_nans, void* workspace, void* stream) {
  if (n < 0) return fail(BSMM_E_ARG, "bsmm_adafactor: n = %d", n);
  if (n && (!grads || !grad_dtypes || !params || !cvs || !rows || !cols))
    return fail(BSMM_E_ARG, "bsmm_adafactor: null array");
  bool any = false;
  for (int i = 0; i < n; ++i) {
    const long long C = rows[i], K = cols[i];
    if (C < 0 || K < 0) return fail(BSMM_E_ARG, "bsmm_adafactor: tensor %d has shape (%lld, %lld)", i, C, K);
    if (!dense_dtype_ok(grad_dtypes[i]))
      return fail(BSMM_E_ARG, "bsmm_adafactor: tensor %d has unsupported grad dtype code %d", i, grad_dtypes[i]);
    if (C > 1 && K > LLONG_MAX / C) return fail(BSMM_E_ARG, "bsmm_adafactor: tensor %d: (%lld, %lld) overflows", i, C, K);
    if (C * K == 0) continue;
    if (af_tiles(C, K) > 0x7fffffffLL || (C > 1 && (C + K + AF_FIN - 1) / AF_FIN > 0x7fffffffLL))
      return fail(BSMM_E_LIMIT, "bsmm_adafactor: tensor %d of (%lld, %lld) exceeds the grid", i, C, K);
    if (!grads[i] || !params[i] || !cvs[i] || (C > 1 && (!rvs || !rvs[i])))
      return fail(BSMM_E_ARG, "bsmm_adafactor: tensor %d has a null pointer", i);
    any = true;
  }
  if (!any) return 0;
  if (!workspace) return fail(BSMM_E_ARG, "bsmm_adafactor: null workspace");
  const AfConsts k = {norm_scale, static_cast<float*>(workspace), lr, decay, epsilon, grad_scale, clip_thresh, saturate,
                      zero_infs, zero_nans};
  const cudaStream_t s = (cudaStream_t)stream;
  return af_for_launches(n, rows, cols,
      [&](int i, AfTensor& t) {
        t.g = grads[i]; t.p = params[i]; t.cv = cvs[i]; t.rv = rows[i] > 1 ? rvs[i] : nullptr;
        t.dtype = (uint8_t)grad_dtypes[i];
        t.vec = aligned16(t.g) && aligned16(t.p) && aligned16(t.cv) && (rows[i] == 1 || cols[i] % 4 == 0);
      },
      [&](const AfTable& tab, int tiles, int fins) {
        mt_adafactor_stats<<<tiles, AF_THREADS, 0, s>>>(tab, k);
        if (int e = check_launch("mt_adafactor_stats")) return e;
        if (fins) {
          mt_adafactor_finish<<<fins, AF_FIN, 0, s>>>(tab, k);
          if (int e = check_launch("mt_adafactor_finish")) return e;
          mt_adafactor_sumsq<<<tiles, AF_THREADS, 0, s>>>(tab, k);
          if (int e = check_launch("mt_adafactor_sumsq")) return e;
        }
        mt_adafactor_rate<<<tab.n, AF_THREADS, 0, s>>>(tab, k);
        if (int e = check_launch("mt_adafactor_rate")) return e;
        mt_adafactor_apply<<<tiles, AF_THREADS, 0, s>>>(tab, k);
        return check_launch("mt_adafactor_apply");
      });
}
static int q_format_args(const char* what, int ebits, int fbits, int denorm) {
  if (ebits < 1 || ebits > 8) return fail(BSMM_E_ARG, "%s: ebits %d outside 1..8", what, ebits);
  if (fbits < 0 || fbits > 23) return fail(BSMM_E_ARG, "%s: fbits %d outside 0..23", what, fbits);
  if (denorm != 0 && denorm != 1) return fail(BSMM_E_ARG, "%s: denorm %d (0 or 1)", what, denorm);
  return 0;
}

// Checks tensor i of a multi-tensor quantize entry: size >= 0, a grid that fits, non-null pointers when not empty.
static int q_check(const char* what, int i, long long size, const void* const* ptrs, int nptr) {
  if (size < 0) return fail(BSMM_E_ARG, "%s: tensor %d has negative size %lld", what, i, size);
  if (q_chunks(size) > 0x7fffffffLL) return fail(BSMM_E_LIMIT, "%s: tensor %d of %lld elements exceeds the grid", what, i, size);
  if (size == 0) return 0;
  for (int j = 0; j < nptr; ++j)
    if (!ptrs[j]) return fail(BSMM_E_ARG, "%s: tensor %d has a null pointer", what, i);
  return 0;
}

int bsmm_quantize(int n, int dtype, const void* const* xs, void* const* ys, long long* const* exps, const long long* sizes,
                  int ebits, int fbits, int denorm, int stochastic, long long* entropy, void* stream) {
  if (n < 0) return fail(BSMM_E_ARG, "bsmm_quantize: n = %d", n);
  if (dtype != BSMM_F32 && dtype != BSMM_BF16) return fail(BSMM_E_ARG, "bsmm_quantize: dtype %d (F32 or BF16)", dtype);
  if (int e = q_format_args("bsmm_quantize", ebits, fbits, denorm)) return e;
  if (dtype == BSMM_BF16 && fbits > 7) return fail(BSMM_E_ARG, "bsmm_quantize: bf16 holds at most 7 fraction bits, got %d", fbits);
  if (stochastic < 0 || stochastic > 2) return fail(BSMM_E_ARG, "bsmm_quantize: stochastic %d (0, 1 or 2)", stochastic);
  if (stochastic && !entropy) return fail(BSMM_E_ARG, "bsmm_quantize: stochastic rounding without an entropy state");
  if (n && (!xs || !ys || !exps || !sizes)) return fail(BSMM_E_ARG, "bsmm_quantize: null array");
  bool any = false;
  for (int i = 0; i < n; ++i) {
    const void* ptrs[3] = {xs[i], ys[i], exps[i]};
    if (int e = q_check("bsmm_quantize", i, sizes[i], ptrs, 3)) return e;
    any = any || sizes[i] > 0;
  }
  if (!any) return 0;
  const QConsts k = {entropy, ebits, fbits, denorm, stochastic ? 1 : 0};
  const cudaStream_t s = (cudaStream_t)stream;
  if (int e = q_for_launches(n, sizes,
          [&](int i, QTensor& t) {
            t.x = xs[i]; t.y = ys[i]; t.exp = exps[i];
            t.vec = aligned16(t.x) && aligned16(t.y);
          },
          [&](const QTable& tab, int chunks, long long) {
            if (dtype == BSMM_F32) {
              if (k.stoch) q_quantize<float, true><<<chunks, Q_THREADS, 0, s>>>(tab, k);
              else         q_quantize<float, false><<<chunks, Q_THREADS, 0, s>>>(tab, k);
            } else {
              if (k.stoch) q_quantize<__nv_bfloat16, true><<<chunks, Q_THREADS, 0, s>>>(tab, k);
              else         q_quantize<__nv_bfloat16, false><<<chunks, Q_THREADS, 0, s>>>(tab, k);
            }
            return check_launch(k.stoch ? "quantize_stochastic" : "quantize");
          }))
    return e;
  if (!k.stoch) return 0;
  q_advance<<<1, 1, 0, s>>>(entropy, (long long)n);
  return check_launch("quantize_stochastic");
}

size_t bsmm_quantize_stats_workspace_bytes(int n, const long long* sizes) {
  if (n < 0 || (n && !sizes)) return 0;
  long long chunks = 0;
  for (int i = 0; i < n; ++i) {
    if (sizes[i] < 0) return 0;
    chunks += q_chunks(sizes[i]);
  }
  return (size_t)chunks * sizeof(QPart);
}

int bsmm_quantize_stats(int n, int dtype, const void* const* xs, const long long* sizes, long long* const* exps,
                        float* stats, int ebits, int fbits, int denorm, int mode, int bias_pad, float stdv_mul,
                        float sat_val, float ftz_val, void* workspace, void* stream) {
  if (n < 0) return fail(BSMM_E_ARG, "bsmm_quantize_stats: n = %d", n);
  if (!dense_dtype_ok(dtype)) return fail(BSMM_E_ARG, "bsmm_quantize_stats: unsupported dtype code %d", dtype);
  if (exps) {
    if (int e = q_format_args("bsmm_quantize_stats", ebits, fbits, denorm)) return e;
    if (mode != 0 && mode != 1) return fail(BSMM_E_ARG, "bsmm_quantize_stats: mode %d (0 or 1)", mode);
  }
  if (n && (!xs || !sizes)) return fail(BSMM_E_ARG, "bsmm_quantize_stats: null array");
  long long total = 0;
  for (int i = 0; i < n; ++i) {
    const void* ptrs[2] = {xs[i], exps ? exps[i] : xs[i]};
    if (int e = q_check("bsmm_quantize_stats", i, sizes[i], ptrs, 2)) return e;
    total += q_chunks(sizes[i]);
  }
  if (total == 0) return 0;
  if (!stats || !workspace) return fail(BSMM_E_ARG, "bsmm_quantize_stats: null stats or workspace");
  QStatConsts k = {stats, workspace, sat_val, ftz_val, stdv_mul, ebits, fbits, denorm, mode, bias_pad, dtype == BSMM_F16};
  const cudaStream_t s = (cudaStream_t)stream;
  QPart* parts = static_cast<QPart*>(workspace);
  return q_for_launches(n, sizes,
      [&](int i, QTensor& t) {
        t.x = xs[i]; t.exp = exps ? exps[i] : nullptr;
        t.vec = aligned16(t.x);
      },
      [&](const QTable& tab, int chunks, long long base) {
        BSMM_DISPATCH_DTYPE(dtype, T, { q_stats<T><<<chunks, Q_THREADS, 0, s>>>(tab, k, parts + base); });
        if (int e = check_launch("quantize_stats")) return e;
        q_stats_finish<<<tab.n, Q_THREADS, 0, s>>>(tab, k, parts + base);
        return check_launch("quantize_stats");
      });
}
// ---- block-sparse convolution (csrc/conv.cuh) ------------------------------------------------------------------------
static bool conv_pair_ok(int a, int b) {
  return dense_dtype_ok(a) && dense_dtype_ok(b) && !((a == BSMM_F16 && b == BSMM_BF16) || (a == BSMM_BF16 && b == BSMM_F16));
}

// Instantiates body with TA / TB for every supported (a, b) dtype pair (fp16 never meets bf16).
#define BSMM_CONV_PAIR(a, b, TA, TB, ...)                                                                               \
  BSMM_DISPATCH_DTYPE(a, TA, {                                                                                        \
    if ((b) == BSMM_F32) { using TB = float; __VA_ARGS__; }                                                           \
    else if ((b) == BSMM_F16 && (a) != BSMM_BF16) { using TB = __half; __VA_ARGS__; }                                 \
    else if ((b) == BSMM_BF16 && (a) != BSMM_F16) { using TB = __nv_bfloat16; __VA_ARGS__; }                          \
  })

static int conv_common_args(const char* what, const int32_t* blocks, const int32_t* channels, const int32_t* lut,
                            int trs, const void* x, const void* f, const void* y, long long N, int C_in, long long P_in,
                            int C_out, long long P_out, int max_out) {
  if (!blocks || !channels || !lut || !x || !f || !y) return fail(BSMM_E_ARG, "%s: null pointer", what);
  if (N < 0 || C_in <= 0 || C_out <= 0 || P_in <= 0 || P_out <= 0 || trs <= 0 || max_out <= 0)
    return fail(BSMM_E_ARG, "%s: bad sizes (N %lld, C_in %d, P_in %lld, C_out %d, P_out %lld, trs %d, max_out %d)", what, N,
                C_in, P_in, C_out, P_out, trs, max_out);
  if (P_out * trs > INT_MAX || P_in > INT_MAX)
    return fail(BSMM_E_LIMIT, "%s: %lld output positions x %d taps exceed the int32 spatial table", what, P_out, trs);
  // xprop puts the 64-row tiles of N * P_out on grid.x (at most 2^31 - 1 CTAs)
  if (N > ((1LL << 37) - 64) / P_out)
    return fail(BSMM_E_LIMIT, "%s: N * P_out = %lld x %lld reaches 2^37 rows", what, N, P_out);
  return 0;
}

int bsmm_conv_xprop(int x_dtype, int f_dtype, const int32_t* blocks, const int* pass_offsets, int passes, int max_out,
                    const int32_t* channels, const int32_t* lut, int trs, const void* x, const void* f, void* y, float* acc,
                    long long N, int C_in, long long P_in, int C_out, long long P_out, int flags, void* stream) {
  const char* what = "bsmm_conv_xprop";
  if (!conv_pair_ok(x_dtype, f_dtype)) return fail(BSMM_E_ARG, "%s: dtype pair (%d, %d)", what, x_dtype, f_dtype);
  if (int e = conv_common_args(what, blocks, channels, lut, trs, x, f, y, N, C_in, P_in, C_out, P_out, max_out)) return e;
  if (passes <= 0 || !pass_offsets) return fail(BSMM_E_ARG, "%s: %d passes", what, passes);
  for (int i = 0; i < passes; ++i)
    if (pass_offsets[i] < 0 || pass_offsets[i + 1] <= pass_offsets[i]) return fail(BSMM_E_ARG, "%s: pass %d is empty", what, i);
  const int col_tiles = (max_out + CONV_T - 1) / CONV_T;
  const long long rows = N * P_out, row_tiles = (rows + CONV_T - 1) / CONV_T;
  for (int i = 0; i < passes; ++i)
    if ((long long)(pass_offsets[i + 1] - pass_offsets[i]) * col_tiles > 65535)
      return fail(BSMM_E_LIMIT, "%s: pass %d has %d blocks of up to %d outputs (at most 65535 64-wide column tiles)", what,
                  i, pass_offsets[i + 1] - pass_offsets[i], max_out);
  const bool multi = passes > 1, y32 = x_dtype == BSMM_F32;
  if (multi && !y32 && !acc) return fail(BSMM_E_ARG, "%s: %d passes into a 16-bit output need an fp32 accumulator", what, passes);
  if (rows == 0) return 0;
  const bool tc = !(flags & BSMM_FLAG_FORCE_GENERIC) && x_dtype == f_dtype && x_dtype != BSMM_F32;
  const cudaStream_t s = (cudaStream_t)stream;
  float* accum = multi ? (y32 ? static_cast<float*>(y) : acc) : nullptr;
  const long long out_elems = N * C_out * P_out;
  if (accum && cudaMemsetAsync(accum, 0, out_elems * sizeof(float), s) != cudaSuccess) return check_launch(what);
  ConvArgs a = {nullptr, channels, lut, x, f, accum ? (void*)accum : y, N, P_in, P_out, rows, C_in, C_out, trs,
                col_tiles, 0, accum ? 1 : 0, 0};
  const char* name = tc ? "wgmma_conv_xprop" : "fma_conv_xprop";
  for (int i = 0; i < passes; ++i) {
    a.blk = reinterpret_cast<const ConvBlk*>(blocks) + pass_offsets[i];
    const dim3 grid((unsigned)row_tiles, (unsigned)((pass_offsets[i + 1] - pass_offsets[i]) * col_tiles));
    if (tc) {
      if (x_dtype == BSMM_BF16) conv_tc_kernel<true, XpropOp<__nv_bfloat16, __nv_bfloat16, CONV_TC_BK>><<<grid, 128, 0, s>>>(a);
      else conv_tc_kernel<false, XpropOp<__half, __half, CONV_TC_BK>><<<grid, 128, 0, s>>>(a);
    } else {
      BSMM_CONV_PAIR(x_dtype, f_dtype, TX, TF, { conv_fma_kernel<XpropOp<TX, TF, 16>><<<grid, 256, 0, s>>>(a); });
    }
    if (int e = check_launch(name)) return e;
  }
  if (multi && !y32) {
    if (int e = launch_float_cast(BSMM_F32, x_dtype, acc, y, out_elems, aligned16(acc) && aligned16(y), s)) return e;
    kernel_name_slot() = name;
  }
  return 0;
}

size_t bsmm_conv_updat_workspace_bytes(long long rows, long long size_f) {
  if (rows < 0 || size_f < 0) return 0;
  return (size_t)((rows + CONV_CHUNK - 1) / CONV_CHUNK) * (size_t)size_f * sizeof(float);
}

int bsmm_conv_updat(int e_dtype, int x_dtype, int f_dtype, const int32_t* blocks, int n_blocks, int max_out, int max_red,
                    const int32_t* channels, const int32_t* lut, int trs, const void* e, const void* x, void* df,
                    float* workspace, long long N, int C_in, long long P_in, int C_out, long long P_out, long long size_f,
                    int flags, void* stream) {
  const char* what = "bsmm_conv_updat";
  if (!conv_pair_ok(e_dtype, x_dtype) || !dense_dtype_ok(f_dtype))
    return fail(BSMM_E_ARG, "%s: dtypes (%d, %d, %d)", what, e_dtype, x_dtype, f_dtype);
  if (int r = conv_common_args(what, blocks, channels, lut, trs, x, e, df, N, C_in, P_in, C_out, P_out, max_out)) return r;
  if (n_blocks <= 0 || max_red <= 0 || size_f <= 0 || size_f > INT_MAX)
    return fail(size_f > INT_MAX ? BSMM_E_LIMIT : BSMM_E_ARG, "%s: %d blocks, max_red %d, size_f %lld", what, n_blocks,
                max_red, size_f);
  const long long rows = N * P_out, chunks = (rows + CONV_CHUNK - 1) / CONV_CHUNK;
  const int row_tiles = (max_out + CONV_T - 1) / CONV_T, col_tiles = (int)(((long long)max_red * trs + CONV_T - 1) / CONV_T);
  if (chunks > 65535) return fail(BSMM_E_LIMIT, "%s: %lld rows exceed 65535 chunks of %d", what, rows, CONV_CHUNK);
  if ((long long)n_blocks * row_tiles * col_tiles > INT_MAX) return fail(BSMM_E_LIMIT, "%s: too many tiles", what);
  if (rows > 0 && !workspace) return fail(BSMM_E_ARG, "%s: null workspace", what);
  const cudaStream_t s = (cudaStream_t)stream;
  const bool tc = !(flags & BSMM_FLAG_FORCE_GENERIC) && e_dtype == x_dtype && x_dtype != BSMM_F32;
  const char* name = tc ? "wgmma_conv_updat" : "fma_conv_updat";
  if (rows > 0) {
    const ConvArgs a = {reinterpret_cast<const ConvBlk*>(blocks), channels, lut, x, e, workspace, N, P_in, P_out, rows,
                        C_in, C_out, trs, col_tiles, row_tiles, 0, size_f};
    const dim3 grid((unsigned)(n_blocks * row_tiles * col_tiles), (unsigned)chunks);
    if (tc) {
      if (x_dtype == BSMM_BF16) conv_tc_kernel<true, UpdatOp<__nv_bfloat16, __nv_bfloat16, CONV_TC_BK>><<<grid, 128, 0, s>>>(a);
      else conv_tc_kernel<false, UpdatOp<__half, __half, CONV_TC_BK>><<<grid, 128, 0, s>>>(a);
    } else {
      BSMM_CONV_PAIR(e_dtype, x_dtype, TE, TX, { conv_fma_kernel<UpdatOp<TE, TX, 16>><<<grid, 256, 0, s>>>(a); });
    }
    if (int r = check_launch(name)) return r;
  }
  const int grid = (int)((size_f + 255) / 256 < 4096 ? (size_f + 255) / 256 : 4096);
  BSMM_DISPATCH_DTYPE(f_dtype, TF, {
    conv_updat_reduce<TF><<<grid, 256, 0, s>>>(workspace, static_cast<TF*>(df), size_f, rows > 0 ? (int)chunks : 0);
  });
  if (int r = check_launch(name)) return r;
  return 0;
}

int bsmm_conv_l2_normalize(int x_dtype, int y_dtype, const int32_t* rows, int n_rows, int trs, const void* x,
                           const float* gain, void* y, float* sum_sqr, float epsilon, void* stream) {
  if (!dense_dtype_ok(x_dtype) || (y_dtype != x_dtype && y_dtype != BSMM_F32))
    return fail(BSMM_E_ARG, "bsmm_conv_l2_normalize: dtypes (%d, %d): y is x's dtype or fp32", x_dtype, y_dtype);
  if (!rows || !x || !y || !sum_sqr || n_rows <= 0 || trs <= 0 || !(epsilon >= 0.f))
    return fail(BSMM_E_ARG, "bsmm_conv_l2_normalize: bad arguments");
  const cudaStream_t s = (cudaStream_t)stream;
  const auto* r = reinterpret_cast<const ConvNormRow*>(rows);
  const int grid = (n_rows + CN_WARPS - 1) / CN_WARPS;
  BSMM_DISPATCH_DTYPE(x_dtype, T, {
    if (y_dtype == BSMM_F32) conv_l2n_kernel<T, float><<<grid, 32 * CN_WARPS, 0, s>>>(r, n_rows, trs, (const T*)x, gain, (float*)y, sum_sqr, epsilon);
    else                     conv_l2n_kernel<T, T><<<grid, 32 * CN_WARPS, 0, s>>>(r, n_rows, trs, (const T*)x, gain, (T*)y, sum_sqr, epsilon);
  });
  return check_launch("conv_l2_normalize");
}

int bsmm_conv_l2_normalize_grad(int x_dtype, int dy_dtype, const int32_t* rows, int n_rows, int trs, const void* dy,
                                const void* x, const float* gain, const float* sum_sqr, void* dx, float* dgain,
                                float epsilon, void* stream) {
  if (!dense_dtype_ok(x_dtype) || (dy_dtype != x_dtype && dy_dtype != BSMM_F32))
    return fail(BSMM_E_ARG, "bsmm_conv_l2_normalize_grad: dtypes (%d, %d): dy is x's dtype or fp32", x_dtype, dy_dtype);
  if (!rows || !dy || !x || !sum_sqr || !dx || n_rows <= 0 || trs <= 0 || !(epsilon >= 0.f))
    return fail(BSMM_E_ARG, "bsmm_conv_l2_normalize_grad: bad arguments");
  const cudaStream_t s = (cudaStream_t)stream;
  const auto* r = reinterpret_cast<const ConvNormRow*>(rows);
  const int grid = (n_rows + CN_WARPS - 1) / CN_WARPS;
  BSMM_DISPATCH_DTYPE(x_dtype, T, {
    if (dy_dtype == BSMM_F32) conv_l2n_grad_kernel<T, float><<<grid, 32 * CN_WARPS, 0, s>>>(r, n_rows, trs, (const float*)dy, (const T*)x, gain, sum_sqr, (T*)dx, dgain, epsilon);
    else                      conv_l2n_grad_kernel<T, T><<<grid, 32 * CN_WARPS, 0, s>>>(r, n_rows, trs, (const T*)dy, (const T*)x, gain, sum_sqr, (T*)dx, dgain, epsilon);
  });
  return check_launch("conv_l2_normalize_grad");
}

// ---- conv edge bias and cwise_linear (csrc/conv_bias.cuh) ---------------------------------------------------------------
static int eb_args(const char* what, int dtype, int layout, const int32_t* pos_edge, const int32_t* lut, int edges,
                   int entries, const void* x, const float* g, const void* y, long long N, long long MPQ, int K) {
  if (!dense_dtype_ok(dtype)) return fail(BSMM_E_ARG, "%s: unsupported dtype code %d", what, dtype);
  if (layout != 0 && layout != 1) return fail(BSMM_E_ARG, "%s: layout must be 0 (channels first) or 1, got %d", what, layout);
  if (!pos_edge || !lut || !g || (N > 0 && (!x || !y))) return fail(BSMM_E_ARG, "%s: null pointer", what);
  if (N < 0 || MPQ <= 0 || K <= 0 || edges <= 0 || entries < edges || entries > MPQ)
    return fail(BSMM_E_ARG, "%s: bad sizes (N %lld, MPQ %lld, K %d, edges %d, entries %d)", what, N, MPQ, K, edges, entries);
  if (MPQ > INT_MAX || 2LL * edges + entries > INT_MAX)
    return fail(BSMM_E_LIMIT, "%s: %lld positions exceed the int32 tables", what, MPQ);
  if (edges > 65535) return fail(BSMM_E_LIMIT, "%s: %d edge patterns exceed grid.y", what, edges);
  if (N > LLONG_MAX / MPQ / K) return fail(BSMM_E_LIMIT, "%s: N * MPQ * K overflows", what);
  return 0;
}

int bsmm_edge_bias(int dtype, int layout, const int32_t* pos_edge, const int32_t* lut, int edges, int entries,
                   const void* x, const float* g, const float* b, void* y, long long N, long long MPQ, int K,
                   int inference, void* stream) {
  const char* what = "bsmm_edge_bias";
  if (int e = eb_args(what, dtype, layout, pos_edge, lut, edges, entries, x, g, y, N, MPQ, K)) return e;
  if (!b) return fail(BSMM_E_ARG, "%s: null pointer", what);
  if (inference && x != y) return fail(BSMM_E_ARG, "%s: inference updates x in place: y must be x", what);
  if (N == 0) return 0;
  EbArgs a = {};
  a.x = x; a.y = y; a.pos_edge = pos_edge; a.lut = lut; a.g = g; a.b = b;
  a.n = N * MPQ * K; a.N = N; a.MPQ = MPQ; a.K = K; a.E = edges; a.entries = entries; a.layout = layout;
  const cudaStream_t s = (cudaStream_t)stream;
  const bool vec = aligned16(x) && aligned16(y) && aligned16(pos_edge);
  if (inference) {
    const bool kvec = vec && K % (16 / dtype_size(dtype)) == 0;
    BSMM_DISPATCH_DTYPE(dtype, T, { return launch_edge_bias_inference<T>(a, kvec, s); });
  }
  BSMM_DISPATCH_DTYPE(dtype, T, { return launch_edge_bias<T>(a, vec, "edge_bias", s); });
  return 0;
}

size_t bsmm_edge_bias_grad_workspace_bytes(long long N, int edges, int max_count, int K) {
  if (N < 0 || edges <= 0 || max_count <= 0 || K <= 0) return 0;
  long long R;
  int S;
  eb_chunks(N, max_count, (long long)edges * K, R, S);
  return (size_t)2 * S * edges * (size_t)K * sizeof(float);
}

int bsmm_edge_bias_grad(int dtype, int layout, const int32_t* pos_edge, const int32_t* lut, int edges, int entries,
                        int max_count, const void* dy, const void* x, const float* g, void* dx, float* dg, float* db,
                        float* workspace, long long N, long long MPQ, int K, void* stream) {
  const char* what = "bsmm_edge_bias_grad";
  if (int e = eb_args(what, dtype, layout, pos_edge, lut, edges, entries, dy, g, dx, N, MPQ, K)) return e;
  if ((N > 0 && !x) || !dg || !db) return fail(BSMM_E_ARG, "%s: null pointer", what);
  if (max_count <= 0 || max_count > entries) return fail(BSMM_E_ARG, "%s: max_count %d", what, max_count);
  if ((long long)edges * K > INT_MAX) return fail(BSMM_E_LIMIT, "%s: edges * K = %d * %d exceeds int32", what, edges, K);
  EbArgs a = {};
  a.x = dy; a.x2 = x; a.y = dx; a.pos_edge = pos_edge; a.lut = lut; a.g = g; a.b = nullptr; a.part = workspace;
  a.n = N * MPQ * K; a.N = N; a.MPQ = MPQ; a.K = K; a.E = edges; a.entries = entries; a.layout = layout;
  eb_chunks(N, max_count, (long long)edges * K, a.R, a.S);
  if (a.S > 0 && !workspace) return fail(BSMM_E_ARG, "%s: null workspace", what);
  const bool vec = aligned16(dy) && aligned16(dx) && aligned16(pos_edge);
  BSMM_DISPATCH_DTYPE(dtype, T, { return launch_edge_bias_grad<T>(a, vec, dg, db, (cudaStream_t)stream); });
  return 0;
}

static int cw_args(const char* what, int dtype, const void* x, const float* a, const float* b, long long N, int C,
                   long long DHW) {
  if (!dense_dtype_ok(dtype)) return fail(BSMM_E_ARG, "%s: unsupported dtype code %d", what, dtype);
  if (!x && N > 0) return fail(BSMM_E_ARG, "%s: null pointer", what);
  if (!a && !b) return fail(BSMM_E_ARG, "%s: neither a gain nor a bias", what);
  if (N < 0 || C <= 0 || DHW <= 0) return fail(BSMM_E_ARG, "%s: bad sizes (N %lld, C %d, DHW %lld)", what, N, C, DHW);
  if (N > LLONG_MAX / C / DHW) return fail(BSMM_E_LIMIT, "%s: N * C * DHW overflows", what);
  if (DHW > 1 && (N * DHW + CW_SEG - 1) / CW_SEG > INT_MAX)
    return fail(BSMM_E_LIMIT, "%s: N * DHW = %lld exceeds the grid", what, N * DHW);
  return 0;
}

int bsmm_cwise_linear(int dtype, const void* x, const float* a, const float* b, void* y, long long N, int C,
                      long long DHW, int relu, int swap, void* stream) {
  const char* what = "bsmm_cwise_linear";
  if (int e = cw_args(what, dtype, x, a, b, N, C, DHW)) return e;
  if (!y && N > 0) return fail(BSMM_E_ARG, "%s: null pointer", what);
  if (N == 0) return 0;
  CwArgs c = {};
  c.x = x; c.y = y; c.a = a; c.b = b; c.n = N * C * DHW; c.N = N; c.DHW = DHW; c.C = C; c.relu = relu != 0;
  c.swap = swap != 0;
  const bool vec = aligned16(x) && aligned16(y);
  BSMM_DISPATCH_DTYPE(dtype, T, { return launch_cwise_linear<T>(c, vec, (cudaStream_t)stream); });
  return 0;
}

size_t bsmm_cwise_linear_grad_workspace_bytes(long long N, int C, long long DHW) {
  if (N < 0 || C <= 0 || DHW <= 0) return 0;
  return (size_t)2 * cw_parts(N, C, DHW) * C * sizeof(float);
}

int bsmm_cwise_linear_grad(int dtype, const void* dy, const void* xy, const float* a, const float* b, void* dx,
                           float* da, float* db, void* workspace, long long N, int C, long long DHW, int relu, int swap,
                           void* stream) {
  const char* what = "bsmm_cwise_linear_grad";
  if (int e = cw_args(what, dtype, dy, a, b, N, C, DHW)) return e;
  if (!a != !da || !b != !db) return fail(BSMM_E_ARG, "%s: da is written iff a is given, db iff b is", what);
  const bool rd = a || relu;
  if (rd && N > 0 && (!xy || !dx)) return fail(BSMM_E_ARG, "%s: null x / y or dx", what);
  CwArgs c = {};
  c.x = dy; c.src = xy; c.y = dx; c.a = a; c.b = b; c.part = (float*)workspace; c.n = N * C * DHW; c.N = N;
  c.DHW = DHW; c.C = C; c.relu = relu != 0; c.swap = swap != 0; c.want_a = a != nullptr; c.want_b = b != nullptr;
  c.rp = cw_rows_per_part(N, C);
  c.parts = cw_parts(N, C, DHW);
  if (c.parts > 0 && !workspace) return fail(BSMM_E_ARG, "%s: null workspace", what);
  const int V = 16 / dtype_size(dtype);
  const bool vec = aligned16(dy) && (!rd || (aligned16(xy) && aligned16(dx))) && (DHW == 1 ? C : DHW) % V == 0;
  BSMM_DISPATCH_DTYPE(dtype, T, { return launch_cwise_linear_grad<T>(c, vec, da, db, (cudaStream_t)stream); });
  return 0;
}
// ---- dw_matmul_large_n ------------------------------------------------------------------------------------------
// Workspace of either route the call may take: a 16-bit call whose shape fits the wgmma route still runs the FMA one
// with misaligned pointers or BSMM_FLAG_FORCE_GENERIC.
size_t bsmm_dw_matmul_large_n_workspace_bytes(int dtype, long long N, int C, int K) {
  if (dtype != BSMM_F32 && dtype != BSMM_F16 && dtype != BSMM_BF16) return 0;
  if (N < 0 || C <= 0 || K <= 0) return 0;
  const size_t fma = dense_dw_workspace(N, C, K, false);
  if (!dense_dw_tc_shape(dtype, N, C, K)) return fma;
  const size_t tc = dense_dw_workspace(N, C, K, true);
  return tc > fma ? tc : fma;
}

int bsmm_dw_matmul_large_n(int dtype, const void* x, const void* e, float* u, long long N, int C, int K,
                           void* workspace, int flags, void* stream) {
  const char* what = "bsmm_dw_matmul_large_n";
  if (dtype != BSMM_F32 && dtype != BSMM_F16 && dtype != BSMM_BF16) return fail(BSMM_E_ARG, "%s: bad dtype %d", what, dtype);
  if (N < 0 || C < 0 || K < 0) return fail(BSMM_E_ARG, "%s: negative size (N=%lld, C=%d, K=%d)", what, N, C, K);
  if ((flags & BSMM_FLAG_FORCE_GENERIC) && (flags & BSMM_FLAG_FORCE_TC)) return fail(BSMM_E_ARG, "%s: contradictory flags", what);
  if (flags & BSMM_FLAG_FORCE_TC) {
    if (dtype == BSMM_F32) return fail(BSMM_E_ARG, "%s: no wgmma kernel for fp32 (it runs on CUDA cores, as in the reference)", what);
    if (!dense_dw_tc_shape(dtype, N, C, K))
      return fail(BSMM_E_ARG, "%s: the wgmma kernel needs C %% 8 == 0, K %% 8 == 0 and N < 2^31 (C=%d, K=%d, N=%lld)", what, C, K, N);
  }
  if (C == 0 || K == 0) return 0;
  if (!u) return fail(BSMM_E_ARG, "%s: null u", what);
  cudaStream_t s = (cudaStream_t)stream;
  if (N == 0) {
    cudaError_t err = cudaMemsetAsync(u, 0, (size_t)C * K * sizeof(float), s);
    if (err != cudaSuccess) { cudaGetLastError(); return fail((int)err, "%s: %s", what, cudaGetErrorString(err)); }
    kernel_name_slot() = "memset_dense_dw";
    return 0;
  }
  if (!x || !e) return fail(BSMM_E_ARG, "%s: null x or e", what);
  const bool aligned = (((uintptr_t)x | (uintptr_t)e) & 15) == 0 && ((uintptr_t)u & 7) == 0 && ((uintptr_t)workspace & 7) == 0;
  bool tc = false;
  if (!(flags & BSMM_FLAG_FORCE_GENERIC) && dense_dw_tc_shape(dtype, N, C, K)) {
    if (!aligned) fail(0, "x and e must be 16-byte aligned, u and the workspace 8-byte aligned, for TMA");
    tc = aligned && wgmma_device();
    if (!tc) {
      if (flags & BSMM_FLAG_FORCE_TC) {
        char why[512];
        snprintf(why, sizeof(why), "%s", err_buf());
        return fail(BSMM_E_ARG, "%s: no wgmma kernel for this call (%s)", what, why);
      }
      note_fallback(what, dtype);
    }
  } else if (dtype != BSMM_F32 && !(flags & BSMM_FLAG_FORCE_GENERIC)) {
    fail(0, "C and K must be multiples of 8 and N below 2^31");
    note_fallback(what, dtype);
  }
  const DwSplit d = dense_dw_split(N, C, K, tc);
  if (d.tiles * d.S > INT_MAX) return fail(BSMM_E_LIMIT, "%s: more than 2^31 - 1 output tiles", what);
  if (d.S > 1 && !workspace)
    return fail(BSMM_E_ARG, "%s: null workspace (bsmm_dw_matmul_large_n_workspace_bytes gives its size)", what);
  if (!device_info().ok) return fail(BSMM_E_NODEV, "no CUDA device");
  return dense_dw_run(tc, dtype, x, e, u, N, C, K, (float*)workspace, s);
}
// ---- fp8 quantisation and xprop ---------------------------------------------------------------------------------
static int fp8_src_ok(int dt) { return dt == BSMM_F32 || dt == BSMM_F16 || dt == BSMM_BF16; }

int bsmm_fp8_quantize(int src_dtype, int fp8_dtype, const void* x, long long n, float* amax, float* scale_inv, void* y,
                      void* stream) {
  const char* what = "bsmm_fp8_quantize";
  if (!fp8_src_ok(src_dtype) || !fp8_code(fp8_dtype))
    return fail(BSMM_E_DTYPE, "%s: needs an fp32 / fp16 / bf16 source and an e4m3 / e5m2 target, got %d -> %d", what, src_dtype, fp8_dtype);
  if (n < 0) return fail(BSMM_E_ARG, "%s: negative size %lld", what, n);
  if (!amax || !scale_inv || (n > 0 && (!x || !y))) return fail(BSMM_E_ARG, "%s: null pointer", what);
  cudaStream_t s = (cudaStream_t)stream;
  uint8_t* q = (uint8_t*)y;
  BSMM_DISPATCH_DTYPE(src_dtype, T, {
    const T* xt = (const T*)x;
    return fp8_dtype == BSMM_E5M2 ? launch_fp8_quantize<T, BSMM_E5M2>(xt, n, amax, scale_inv, q, s)
                                  : launch_fp8_quantize<T, BSMM_E4M3>(xt, n, amax, scale_inv, q, s);
  });
  return 0;
}

int bsmm_fp8_weights(int src_dtype, int fp8_dtype, int bsize, int blocks, const void* w, float* amax, float* scale_inv,
                     void* wq, void* wq_t, void* stream) {
  const char* what = "bsmm_fp8_weights";
  if (bsize != 32 && bsize != 64) return fail(BSMM_E_BSIZE, "%s: fp8 weights need block size 32 or 64, got %d", what, bsize);
  if (!fp8_src_ok(src_dtype) || !fp8_code(fp8_dtype))
    return fail(BSMM_E_DTYPE, "%s: needs an fp32 / fp16 / bf16 source and an e4m3 / e5m2 target, got %d -> %d", what, src_dtype, fp8_dtype);
  if (blocks <= 0) return fail(BSMM_E_ARG, "%s: blocks must be positive, got %d", what, blocks);
  if (!w || !amax || !scale_inv || !wq || !wq_t) return fail(BSMM_E_ARG, "%s: null pointer", what);
  if (((uintptr_t)wq | (uintptr_t)wq_t) & 15) return fail(BSMM_E_ALIGN, "%s: wq and wq_t must be 16-byte aligned", what);
  cudaStream_t s = (cudaStream_t)stream;
  uint8_t *q = (uint8_t*)wq, *qt = (uint8_t*)wq_t;
  BSMM_DISPATCH_DTYPE(src_dtype, T, {
    const T* wt = (const T*)w;
    return fp8_dtype == BSMM_E5M2 ? launch_fp8_weights<T, BSMM_E5M2>(bsize, blocks, wt, amax, scale_inv, q, qt, s)
                                  : launch_fp8_weights<T, BSMM_E4M3>(bsize, blocks, wt, amax, scale_inv, q, qt, s);
  });
  return 0;
}

int bsmm_xprop_fp8(int x_dtype, int w_dtype, int y_dtype, int axis, int bsize, int bprop, const int32_t* lut, int n_out,
                   int n_in, int blocks, const void* x, const void* w, void* y, int N, const float* x_scale_inv,
                   const float* w_scale_inv, void* stream) {
  const char* what = "bsmm_xprop_fp8";
  if (axis != 1) return fail(BSMM_E_BSIZE, "%s: fp8 xprop needs feature axis 1, got %d", what, axis);
  if (bsize != 32 && bsize != 64) return fail(BSMM_E_BSIZE, "%s: fp8 xprop needs block size 32 or 64, got %d", what, bsize);
  if (!fp8_code(x_dtype) || !fp8_code(w_dtype) || (y_dtype != BSMM_F16 && y_dtype != BSMM_BF16))
    return fail(BSMM_E_DTYPE, "%s: needs e4m3 / e5m2 x and w and an fp16 / bf16 y, got x %d, w %d, y %d", what, x_dtype,
                w_dtype, y_dtype);
  if (!lut || !x || !w || !y || !x_scale_inv || !w_scale_inv) return fail(BSMM_E_ARG, "%s: null pointer", what);
  // fprop and bprop run the same kernel: the direction is in the LUT and the weight layout the caller passes
  if (bprop != 0 && bprop != 1) return fail(BSMM_E_ARG, "%s: bprop must be 0 or 1, got %d", what, bprop);
  if (n_out <= 0 || n_in <= 0 || blocks < 0 || N < 0) return fail(BSMM_E_ARG, "%s: bad sizes", what);
  if (n_out >= 65536 || n_in >= 65536) return fail(BSMM_E_LIMIT, "%s: more than 65535 blocks per dimension", what);
  if (((uintptr_t)x | (uintptr_t)w | (uintptr_t)y) & 15) return fail(BSMM_E_ALIGN, "%s: x, w and y must be 16-byte aligned", what);
  if (N == 0) return 0;
  return tc_xprop_fp8(x_dtype, w_dtype, y_dtype, bsize, lut, n_out, n_in, blocks, x, w, y, N, x_scale_inv, w_scale_inv,
                      (cudaStream_t)stream);
}

int bsmm_fp8_quantize_t(int src_dtype, int fp8_dtype, const void* x, long long rows, long long cols, float* amax,
                        float* scale_inv, void* y, void* yt, long long yt_pitch, void* stream) {
  const char* what = "bsmm_fp8_quantize_t";
  if (!fp8_src_ok(src_dtype) || !fp8_code(fp8_dtype))
    return fail(BSMM_E_DTYPE, "%s: needs an fp32 / fp16 / bf16 source and an e4m3 / e5m2 target, got %d -> %d", what, src_dtype, fp8_dtype);
  if (rows < 0 || cols < 0) return fail(BSMM_E_ARG, "%s: negative size %lld x %lld", what, rows, cols);
  if (!amax || !scale_inv || (!y && !yt)) return fail(BSMM_E_ARG, "%s: null pointer", what);
  if (rows * cols > 0 && !x) return fail(BSMM_E_ARG, "%s: null pointer", what);
  if (yt) {
    if (yt_pitch < rows) return fail(BSMM_E_ARG, "%s: yt_pitch %lld below rows %lld", what, yt_pitch, rows);
    if (yt_pitch % 16) return fail(BSMM_E_ALIGN, "%s: yt_pitch %lld is not a multiple of 16", what, yt_pitch);
    if ((uintptr_t)yt & 3) return fail(BSMM_E_ALIGN, "%s: yt must be 4-byte aligned", what);
  }
  cudaStream_t s = (cudaStream_t)stream;
  uint8_t *q = (uint8_t*)y, *qt = (uint8_t*)yt;
  BSMM_DISPATCH_DTYPE(src_dtype, T, {
    const T* xt = (const T*)x;
    return fp8_dtype == BSMM_E5M2 ? launch_fp8_quantize_t<T, BSMM_E5M2>(xt, rows, cols, amax, scale_inv, q, qt, yt_pitch, s)
                                  : launch_fp8_quantize_t<T, BSMM_E4M3>(xt, rows, cols, amax, scale_inv, q, qt, yt_pitch, s);
  });
  return 0;
}

int bsmm_updat_fp8(int x_dtype, int dy_dtype, int dw_dtype, int bsize, int blocks, int n_c_blocks, int n_k_blocks,
                   const void* const* xts, const void* const* dyts, const float* const* x_scale_invs,
                   const float* const* dy_scale_invs, int pcount, void* dw, long long N, long long pitch, float beta,
                   const int32_t* sched, int sched_tiles, int sched_tile_blocks, void* stream) {
  const char* what = "bsmm_updat_fp8";
  if (bsize != 32 && bsize != 64) return fail(BSMM_E_BSIZE, "%s: fp8 updat needs block size 32 or 64, got %d", what, bsize);
  if (!fp8_code(x_dtype) || !fp8_code(dy_dtype) || !fp8_src_ok(dw_dtype))
    return fail(BSMM_E_DTYPE, "%s: needs e4m3 / e5m2 xt and dyt and an fp32 / fp16 / bf16 dw, got xt %d, dyt %d, dw %d", what,
                x_dtype, dy_dtype, dw_dtype);
  if (pcount < 1 || pcount > BSMM_MAX_PAIRS)
    return fail(BSMM_E_ARG, "%s: pcount must be in [1,%d], got %d", what, BSMM_MAX_PAIRS, pcount);
  if (!xts || !dyts || !x_scale_invs || !dy_scale_invs || !dw || !sched) return fail(BSMM_E_ARG, "%s: null pointer", what);
  for (int i = 0; i < pcount; ++i)
    if (!xts[i] || !dyts[i] || !x_scale_invs[i] || !dy_scale_invs[i]) return fail(BSMM_E_ARG, "%s: null pointer in pair %d", what, i);
  if (N < 0) return fail(BSMM_E_ARG, "%s: negative N %lld", what, N);
  if (pitch < N) return fail(BSMM_E_ARG, "%s: pitch %lld below N %lld", what, pitch, N);
  if (pitch % 16) return fail(BSMM_E_ALIGN, "%s: pitch %lld is not a multiple of 16", what, pitch);
  if (beta != 0.f && beta != 1.f) return fail(BSMM_E_ARG, "%s: beta must be 0 or 1", what);
  if (blocks <= 0 || n_c_blocks <= 0 || n_k_blocks <= 0 || sched_tiles <= 0) return fail(BSMM_E_ARG, "%s: bad sizes", what);
  if (sched_tile_blocks != 256 / bsize)
    return fail(BSMM_E_ARG, "%s: schedule built for %d slots per tile, kernel needs %d", what, sched_tile_blocks, 256 / bsize);
  if (N > INT_MAX) return fail(BSMM_E_LIMIT, "%s: N above 2^31 - 1", what);
  if ((uintptr_t)dw & 15) return fail(BSMM_E_ALIGN, "%s: dw must be 16-byte aligned", what);
  for (int i = 0; i < pcount; ++i)
    if (((uintptr_t)xts[i] | (uintptr_t)dyts[i]) & 15) return fail(BSMM_E_ALIGN, "%s: xt and dyt must be 16-byte aligned", what);
  cudaStream_t s = (cudaStream_t)stream;
  if (N == 0) {                                        // as bsmm_updat: an empty sum, so dw = 0 (beta 0) or unchanged
    if (beta != 0.f) return 0;
    const size_t bytes = (size_t)blocks * bsize * bsize * (dw_dtype == BSMM_F32 ? 4 : 2);
    cudaError_t e = cudaMemsetAsync(dw, 0, bytes, s);
    if (e != cudaSuccess) { cudaGetLastError(); return fail((int)e, "%s: %s", what, cudaGetErrorString(e)); }
    return 0;
  }
  return tc_updat_fp8(x_dtype, dy_dtype, dw_dtype, bsize, n_c_blocks, n_k_blocks, xts, dyts, x_scale_invs, dy_scale_invs,
                      pcount, dw, N, pitch, beta != 0.f ? 1 : 0, sched, sched_tiles, s);
}
}  // extern "C"
