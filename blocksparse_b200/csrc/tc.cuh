// Warpgroup-MMA (wgmma, sm_90a) kernel families.
//
// tc_xprop: block-sparse fprop / bprop for 16-bit dtypes, both feature axes, block size 16 / 32 / 64.
//   Replaces hgemm_blocksparse_64x64x64_nx_dsd / 64x32x32_nx_dsd
//   (reference src/blocksparse_hgemm_nc_op_gpu.cu:38-551) and the feature-axis-0 family
//   hgemm_blocksparse_xn_64_sdd (src/blocksparse_hgemm_cn_64_op_gpu.cu:9-717).
//
// Formulation (see DESIGN.md "xprop on wgmma"): one CTA (one warpgroup) owns one output block of 128 minibatch
// rows.  The minibatch sits on the MMA M axis (two m64 wgmma per K=16 step), the output block's BS features on N,
// and the CTA walks its LUT row: every entry is an (activation tile, W block) pair that TMA stages into a ring of
// shared-memory buffers, each completing on one mbarrier, while the warpgroup multiplies the previous entries.
// Accumulation is in fp32 registers in LUT order, so results are deterministic.
//   fprop: B = W[c][k] read as K x N with N contiguous (MN-major);  bprop: B = W[c][k] as N x K (K-major).
//   axis 1: A = X[n][c] tile (K-major);  axis 0: A = X[c][n] tile read transposed (MN-major).
// CL = 2 (pair tiles, 32 x 32 blocks): thread-block clusters of two CTAs on neighbouring minibatch tiles of the same
// output block.  Both walk the same LUT row, so each W block is fetched once by one of them (alternating) and delivered
// to both by TMA multicast; the accumulation order is unchanged, so results are bit-identical to CL = 1.
#pragma once
#include <cuda.h>
#include "common.cuh"
#include "ptx.cuh"

namespace bsmm {
constexpr int TC_NOT_APPLICABLE = -1000;

// ---- TMA descriptor encoding via the driver entry point (no -lcuda link dependency) -----------
typedef CUresult (*TmapEncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                 const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                 CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
inline TmapEncodeFn tmap_encoder() {
  static TmapEncodeFn fn = []() -> TmapEncodeFn {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess) return nullptr;
    return (TmapEncodeFn)p;
  }();
  return fn;
}
// Element size of a tensor-map dtype code: 1 byte for the fp8 codes, 2 for fp16 / bf16.
inline uint64_t tmap_elem_bytes(int dtype) { return dtype == BSMM_E4M3 || dtype == BSMM_E5M2 ? 1 : 2; }
// 2-D row-major tensor [outer][inner] of 16-bit (fp16 / bf16) or 1-byte (fp8, encoded as UINT8) elements;
// box = box_outer rows x box_inner elements.
inline int make_tmap_2d(CUtensorMap* m, int dtype, const void* base, uint64_t inner, uint64_t outer, uint64_t row_pitch_elems,
                        uint32_t box_inner, uint32_t box_outer, CUtensorMapSwizzle swz) {
  TmapEncodeFn enc = tmap_encoder();
  if (!enc) return fail(BSMM_E_NODEV, "cuTensorMapEncodeTiled entry point not available");
  const uint64_t esize = tmap_elem_bytes(dtype);
  cuuint64_t dims[2] = {inner, outer};
  cuuint64_t strides[1] = {row_pitch_elems * esize};
  cuuint32_t box[2] = {box_inner, box_outer};
  cuuint32_t estr[2] = {1, 1};
  CUtensorMapDataType dt = esize == 1 ? CU_TENSOR_MAP_DATA_TYPE_UINT8
                           : dtype == BSMM_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
  CUresult r = enc(m, dt, 2, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swz,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(BSMM_E_ARG, "cuTensorMapEncodeTiled failed with CUresult %d", (int)r);
  return 0;
}

// Encoding a CUtensorMap costs a few microseconds of host time and the same (pointer, shape) tuples come back every
// training step, so the encoded descriptors are kept in a small thread-local cache (round-robin replacement).  The
// descriptors are still passed to the kernels by value (__grid_constant__), so launches stay CUDA-graph capturable.
struct TmapKey {
  const void* base; uint64_t inner, outer, pitch; uint32_t box_inner, box_outer; int dtype, swz, dev;
  bool operator==(const TmapKey& o) const {
    return base == o.base && inner == o.inner && outer == o.outer && pitch == o.pitch && box_inner == o.box_inner &&
           box_outer == o.box_outer && dtype == o.dtype && swz == o.swz && dev == o.dev;
  }
};
constexpr int TMAP_CACHE_SLOTS = 32;
struct TmapCache { TmapKey key[TMAP_CACHE_SLOTS]; CUtensorMap map[TMAP_CACHE_SLOTS]; int used = 0, next = 0; };
inline int cached_tmap_2d(CUtensorMap* m, int dtype, const void* base, uint64_t inner, uint64_t outer, uint64_t row_pitch_elems,
                          uint32_t box_inner, uint32_t box_outer, CUtensorMapSwizzle swz) {
  static thread_local TmapCache cache;
  int dev = 0;
  cudaGetDevice(&dev);
  const TmapKey k = {base, inner, outer, row_pitch_elems, box_inner, box_outer, dtype, (int)swz, dev};
  for (int i = 0; i < cache.used; ++i)
    if (cache.key[i] == k) { *m = cache.map[i]; return 0; }
  if (int e = make_tmap_2d(m, dtype, base, inner, outer, row_pitch_elems, box_inner, box_outer, swz)) return e;
  const int slot = cache.next;
  cache.key[slot] = k; cache.map[slot] = *m;
  cache.next = (slot + 1) % TMAP_CACHE_SLOTS;
  if (cache.used < TMAP_CACHE_SLOTS) ++cache.used;
  return 0;
}
inline CUtensorMapSwizzle tmap_swizzle_for_row(int row_bytes) {
  return row_bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B : row_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B;
}

// Applicability shared by every wgmma family: an sm_90 device and this host thread bound to its primary context
// (cuTensorMapEncodeTiled is a driver entry point and an autograd worker thread may not have touched CUDA yet).
inline bool wgmma_device() {
  const DeviceInfo& dev = device_info();
  if (!dev.ok || dev.cc_major != 9) { fail(0, "wgmma kernels need an sm_90 device"); return false; }
  static thread_local bool ctx_bound = false;
  if (!ctx_bound) { cudaFree(nullptr); ctx_bound = true; }
  return true;
}

// sticky device-side error word: a kernel whose bounded wait timed out stores a non-zero code here
__device__ int g_tc_error = 0;

// Dynamic shared memory is only guaranteed 16-byte alignment; the swizzled TMA / wgmma tiles need 1024.
constexpr size_t SMEM_ALIGN_SLACK = 1024;
__device__ __forceinline__ uint32_t aligned_smem_base(const void* p) { return (ptx::smem_u32(p) + 1023u) & ~1023u; }

template <bool BF16> __device__ __forceinline__ uint32_t pack2(float a, float b) {
  if constexpr (BF16) { __nv_bfloat162 q = __floats2bfloat162_rn(a, b); return *reinterpret_cast<uint32_t*>(&q); }
  else { __half2 q = __floats2half2_rn(a, b); return *reinterpret_cast<uint32_t*>(&q); }
}
template <bool BF16> __device__ __forceinline__ uint16_t pack1(float a) {
  if constexpr (BF16) { __nv_bfloat16 q = __float2bfloat16_rn(a); return *reinterpret_cast<uint16_t*>(&q); }
  else { __half q = __float2half_rn(a); return *reinterpret_cast<uint16_t*>(&q); }
}

// ---------------------------------------------------------------------------------------------
constexpr int XP_STAGES = 4;          // LUT entries in flight per CTA
constexpr int XP_THREADS = 128;       // one warpgroup
template <int BS> struct XpropShape {
  static constexpr uint32_t XBYTES = 128 * BS * 2;                          // activation tile: 128 minibatch rows x BS features
  static constexpr uint32_t WBYTES = BS * BS * 2;
  static constexpr uint32_t STAGE = (XBYTES + WBYTES + 1023) / 1024 * 1024;
  static constexpr size_t SMEM = XP_STAGES * STAGE + SMEM_ALIGN_SLACK;
};

struct XpropTcParams {
  const int32_t* lut;        // row LUT: [n_out][2] = (first entry, count), entries (W block, input block)
  void* y;
  long long y_pitch;         // elements
  int N;
};
struct XpropTmaps { CUtensorMap x, w; };

template <int BS, bool BF16, bool AXIS0, bool BPROP, int CL = 1>
__global__ void __launch_bounds__(XP_THREADS)
tc_xprop_kernel(const XpropTcParams p, const __grid_constant__ XpropTmaps maps) {
  using Sh = XpropShape<BS>;
  constexpr int ST = XP_STAGES;
  constexpr uint32_t ROW = BS * 2;                         // bytes per row of a W block / axis-1 activation tile
  constexpr uint32_t SWZ = ptx::swz_for_row(ROW);
  extern __shared__ uint8_t smem_raw[];
  __shared__ uint64_t full[ST];
  const uint32_t base = aligned_smem_base(smem_raw);
  const int tid = threadIdx.x, warp = tid / 32, lane = tid % 32;
  const int nt = blockIdx.x, o = blockIdx.y;
  const int first = p.lut[2 * o], count = p.lut[2 * o + 1];
  const int2* ent = reinterpret_cast<const int2*>(p.lut) + first;
  const int crank = CL == 2 ? (int)ptx::cluster_ctarank() : 0;

  auto issue = [&](int e) {                                // one thread: stage entry e
    const int2 wi = ent[e];                                // (W block, input block)
    const uint32_t st = base + (uint32_t)(e % ST) * Sh::STAGE;
    uint64_t* bar = &full[e % ST];
    ptx::mbar_expect_tx(bar, Sh::XBYTES + Sh::WBYTES);
    if (!AXIS0) {
      ptx::tma_load_2d(st, &maps.x, bar, wi.y * BS, nt * 128);                  // [128 n][BS c]
    } else {                                                                    // [BS c][128 n] as two 64-column boxes
      ptx::tma_load_2d(st, &maps.x, bar, nt * 128, wi.y * BS);
      ptx::tma_load_2d(st + Sh::XBYTES / 2, &maps.x, bar, nt * 128 + 64, wi.y * BS);
    }
    if (CL == 1) ptx::tma_load_2d(st + Sh::XBYTES, &maps.w, bar, 0, wi.x * BS);
    else if (e % 2 == crank) ptx::tma_load_2d_mc(st + Sh::XBYTES, &maps.w, bar, 0, wi.x * BS, (uint16_t)3);
  };

  if (tid == 0) {
    for (int i = 0; i < ST; ++i) ptx::mbar_init(&full[i], 1);
    ptx::fence_mbar_init();
    ptx::prefetch_tensormap(&maps.x); ptx::prefetch_tensormap(&maps.w);
  }
  __syncthreads();
  if (CL == 2) ptx::cluster_sync();                        // the peer's barriers exist before anything is multicast to them
  if (tid == 0)
    for (int e = 0; e < count && e < ST; ++e) issue(e);

  float acc[2][BS / 2];
#pragma unroll
  for (int m = 0; m < 2; ++m)
#pragma unroll
    for (int i = 0; i < BS / 2; ++i) acc[m][i] = 0.f;

  for (int e = 0; e < count; ++e) {
    const uint32_t st = base + (uint32_t)(e % ST) * Sh::STAGE;
    if (!ptx::mbar_wait(&full[e % ST], (uint32_t)(e / ST) & 1)) g_tc_error = 1;
    ptx::wg_fence();
#pragma unroll
    for (int ks = 0; ks < BS / 16; ++ks) {
      const uint64_t bdesc = BPROP ? ptx::make_desc(st + Sh::XBYTES + ks * 32, 16, 8 * ROW, SWZ)
                                   : ptx::make_desc(st + Sh::XBYTES + ks * 16 * ROW, Sh::WBYTES, 8 * ROW, SWZ);
#pragma unroll
      for (int m = 0; m < 2; ++m) {
        const uint64_t adesc = AXIS0 ? ptx::make_desc(st + m * (Sh::XBYTES / 2) + ks * 2048, Sh::XBYTES / 2, 1024, ptx::SWZ_128B)
                                     : ptx::make_desc(st + m * 64 * ROW + ks * 32, 16, 8 * ROW, SWZ);
        ptx::wgmma<BF16, AXIS0 ? 1 : 0, BPROP ? 0 : 1, BS>(acc[m], adesc, bdesc);
      }
    }
    ptx::wg_commit();
    ptx::wg_wait<1>();                                     // entry e-1 has been consumed by the whole warpgroup ...
    if (CL == 2) ptx::cluster_sync();                      // ... (and by the peer, whose buffer a multicast also refills)
    else __syncthreads();
    if (tid == 0 && e >= 1 && e - 1 + ST < count) issue(e - 1 + ST);   // ... so its buffer can be refilled
  }
  ptx::wg_wait<0>();
  ptx::wg_fence_regs(acc[0]);
  ptx::wg_fence_regs(acc[1]);
  if (CL == 2) ptx::cluster_sync();                        // nobody leaves while the peer may still multicast into it

  // epilogue (also zero-fills output blocks whose LUT row is empty)
  uint16_t* y = reinterpret_cast<uint16_t*>(p.y);
#pragma unroll
  for (int m = 0; m < 2; ++m)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const long long n = (long long)nt * 128 + m * 64 + warp * 16 + lane / 4 + 8 * h;
      if (n >= p.N) continue;
#pragma unroll
      for (int j = 0; j < BS / 8; ++j) {
        const int col = o * BS + 8 * j + 2 * (lane % 4);
        const float a = acc[m][4 * j + 2 * h], b = acc[m][4 * j + 2 * h + 1];
        if (!AXIS0) {
          *reinterpret_cast<uint32_t*>(y + n * p.y_pitch + col) = pack2<BF16>(a, b);
        } else {
          y[(long long)col * p.y_pitch + n] = pack1<BF16>(a);
          y[(long long)(col + 1) * p.y_pitch + n] = pack1<BF16>(b);
        }
      }
    }
}

template <int BS, bool BF16, bool AXIS0, bool BPROP>
int launch_tc_xprop(const XpropTcParams& p, const XpropTmaps& maps, int n_out, cudaStream_t s) {
  auto kern = tc_xprop_kernel<BS, BF16, AXIS0, BPROP>;
  constexpr size_t smem = XpropShape<BS>::SMEM;
  static thread_local uint64_t configured = 0;
  if (int e = ensure_dyn_smem(kern, smem, configured)) return e;
  kern<<<dim3((unsigned)((p.N + 127) / 128), (unsigned)n_out), XP_THREADS, smem, s>>>(p, maps);
  return check_launch(BS == 16 ? "wgmma_xprop_bs16" : BS == 32 ? "wgmma_xprop_bs32" : "wgmma_xprop_bs64");
}

template <bool BF16, bool AXIS0, bool BPROP>
int launch_tc_xprop_pair(const XpropTcParams& p, const XpropTmaps& maps, int n_out, cudaStream_t s) {
  auto kern = tc_xprop_kernel<32, BF16, AXIS0, BPROP, 2>;
  constexpr size_t smem = XpropShape<32>::SMEM;
  static thread_local uint64_t configured = 0;
  if (int e = ensure_dyn_smem(kern, smem, configured)) return e;
  const unsigned nt = (unsigned)((p.N + 127) / 128);
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((nt + 1) & ~1u, (unsigned)n_out);     // an odd last tile's partner reads zeros and stores nothing
  cfg.blockDim = dim3(XP_THREADS); cfg.dynamicSmemBytes = smem; cfg.stream = s;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = 2; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr; cfg.numAttrs = 1;
  cudaError_t e = cudaLaunchKernelEx(&cfg, kern, p, maps);
  if (e != cudaSuccess) { cudaGetLastError(); return fail((int)e, "cluster launch: %s", cudaGetErrorString(e)); }
  return check_launch("wgmma_xprop_bs32_pair");
}

template <int BS, bool BF16>
int dispatch_tc_xprop(const XpropTcParams& p, const XpropTmaps& maps, int n_out, bool axis0, bool bprop, bool pair, cudaStream_t s) {
  if constexpr (BS == 32) {
    if (pair) {
      if (axis0) return bprop ? launch_tc_xprop_pair<BF16, true, true>(p, maps, n_out, s) : launch_tc_xprop_pair<BF16, true, false>(p, maps, n_out, s);
      return bprop ? launch_tc_xprop_pair<BF16, false, true>(p, maps, n_out, s) : launch_tc_xprop_pair<BF16, false, false>(p, maps, n_out, s);
    }
  }
  if (axis0) return bprop ? launch_tc_xprop<BS, BF16, true, true>(p, maps, n_out, s) : launch_tc_xprop<BS, BF16, true, false>(p, maps, n_out, s);
  return bprop ? launch_tc_xprop<BS, BF16, false, true>(p, maps, n_out, s) : launch_tc_xprop<BS, BF16, false, false>(p, maps, n_out, s);
}

// pair: 32 x 32 blocks only, 2-CTA clusters sharing the W blocks (CL = 2 above)
inline int tc_xprop(int dtype, int axis, int bsize, int bprop, const int32_t* lut, int n_out, int n_in, int blocks,
                    const void* x, const void* w, void* y, int N, const float* gate, bool pair, cudaStream_t s) {
  if (dtype != BSMM_F16 && dtype != BSMM_BF16) { fail(0, "fp32 runs on the FMA path"); return TC_NOT_APPLICABLE; }
  if (bsize != 16 && bsize != 32 && bsize != 64) { fail(0, "block size %d uses the CUDA-core path", bsize); return TC_NOT_APPLICABLE; }
  if (gate != nullptr) { fail(0, "gated xprop uses the CUDA-core path"); return TC_NOT_APPLICABLE; }
  if (axis == 0 && (N & 7)) { fail(0, "feature_axis 0 needs N %% 8 == 0 for TMA (row pitch multiple of 16 bytes)"); return TC_NOT_APPLICABLE; }
  if (((uintptr_t)x | (uintptr_t)w | (uintptr_t)y) & 15) { fail(0, "pointers must be 16-byte aligned for TMA"); return TC_NOT_APPLICABLE; }
  if (!wgmma_device()) return TC_NOT_APPLICABLE;
  if (pair && bsize != 32) return fail(BSMM_E_ARG, "bsmm_xprop: pair tiles need 32 x 32 blocks");

  const uint64_t Cin = (uint64_t)n_in * bsize, Cout = (uint64_t)n_out * bsize;
  const CUtensorMapSwizzle swz = tmap_swizzle_for_row(bsize * 2);
  XpropTmaps maps;
  if (axis == 1) {
    if (int e = cached_tmap_2d(&maps.x, dtype, x, Cin, (uint64_t)N, Cin, bsize, 128, swz)) return e;
  } else {       // (C, N): inner dim = minibatch; box = 64 columns x bs feature rows, 128-byte rows
    if (int e = cached_tmap_2d(&maps.x, dtype, x, (uint64_t)N, Cin, (uint64_t)N, 64, bsize, CU_TENSOR_MAP_SWIZZLE_128B)) return e;
  }
  if (int e = cached_tmap_2d(&maps.w, dtype, w, (uint64_t)bsize, (uint64_t)blocks * bsize, (uint64_t)bsize, bsize, bsize, swz)) return e;

  XpropTcParams p;
  p.lut = lut;
  p.y = y; p.y_pitch = axis == 0 ? (long long)N : (long long)Cout; p.N = N;
  const bool bf = dtype == BSMM_BF16, a0 = axis == 0, bp = bprop != 0;
  if (bsize == 16) return bf ? dispatch_tc_xprop<16, true>(p, maps, n_out, a0, bp, false, s) : dispatch_tc_xprop<16, false>(p, maps, n_out, a0, bp, false, s);
  if (bsize == 32) return bf ? dispatch_tc_xprop<32, true>(p, maps, n_out, a0, bp, pair, s) : dispatch_tc_xprop<32, false>(p, maps, n_out, a0, bp, pair, s);
  return bf ? dispatch_tc_xprop<64, true>(p, maps, n_out, a0, bp, false, s) : dispatch_tc_xprop<64, false>(p, maps, n_out, a0, bp, false, s);
}

}  // namespace bsmm

#include "tc_xprop2.cuh"
#include "tc_updat.cuh"
#include "tc_bst.cuh"
#include "tc_bst_attn.cuh"
#include "tc_bst_attn_bwd.cuh"
