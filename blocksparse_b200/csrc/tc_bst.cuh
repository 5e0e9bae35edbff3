// wgmma kernels for the block-sparse transformer GEMMs, block size 64, 16-bit dense operands.
//   tc_bst_nt_kernel : C[b,h,blk] = A[b, q-blk, h, :] . B[b, k-blk, h, :]^T          (dense . dense^T -> sparse)
//                      replaces bst_hgemm_64x64x64_nt      (reference src/bst_hgemm_op_gpu.cu:651-1098)
//   tc_bst_xn_kernel : C[b, o-blk, h, :] = sum_j op(A[b,h,blk_j]) . B[b, in_j, h, :]   (sparse . dense -> dense)
//                      replaces bst_hgemm_64x64x64_xn<OP_A> (reference src/bst_hgemm_op_gpu.cu:16-646)
//
// Both ops are memory-bound at head_state 64 (~32 flop/B), so the formulation favours simple,
// fully coalesced TMA traffic and many small CTAs in flight over tensor-pipe utilisation.  One warpgroup per CTA:
//   NT: one 64 x 64 score block per CTA: A = the query tile, B = the key tile, both K-major with the head split as a
//       TMA coordinate (column h*head_state), so no transpose kernel exists, as in the reference.
//   XN: one 64-row output block per CTA walking its LUT row through a ring of TMA stages.  NN reads the sparse block
//       K-major, TN reads the same tile MN-major (transpose for free in the descriptor); B is the dense tile, MN-major.
#pragma once
#include <type_traits>
#include "common.cuh"
#include "ptx.cuh"

namespace bsmm {

constexpr int BST_THREADS = 128;
constexpr int BST_STAGES = 4;
constexpr uint32_t BST_TILE = 64 * 64 * 2;   // one 64 x 64 16-bit tile with 128-byte rows (SW128)

// ------------------------------------------------------------------------------------------------
struct BstNtParams {
  const int32_t* lut;       // [lut_heads][blocks][2] = (query block, key block)
  long long lut_head_stride;
  int heads, blocks, head_state;
  int ctx_rows_a, ctx_rows_b;   // rows per batch element of a / b
  void* c;
};
struct BstNtTmaps { CUtensorMap a, b; };

template <bool BF16, typename TC>
__global__ void __launch_bounds__(BST_THREADS)
tc_bst_nt_kernel(const BstNtParams p, const __grid_constant__ BstNtTmaps maps) {
  extern __shared__ uint8_t smem_raw[];
  __shared__ uint64_t full;
  const uint32_t base = aligned_smem_base(smem_raw);          // query chunks at 0 / 8 KB, key chunks at 16 / 24 KB
  const int tid = threadIdx.x, warp = tid / 32, lane = tid % 32;
  const int chunks = p.head_state / 64;
  const int blk = (int)(blockIdx.x % (unsigned)p.blocks);
  const int z = (int)(blockIdx.x / (unsigned)p.blocks);
  const int b = z / p.heads, h = z % p.heads;
  const int32_t* lut = p.lut + h * p.lut_head_stride;
  const int qb = lut[2 * blk], kb = lut[2 * blk + 1];

  if (tid == 0) {
    ptx::mbar_init(&full, 1);
    ptx::fence_mbar_init();
    ptx::mbar_expect_tx(&full, (uint32_t)(2 * chunks) * BST_TILE);
    for (int c = 0; c < chunks; ++c) {
      const int col = h * p.head_state + c * 64;
      ptx::tma_load_2d(base + c * BST_TILE, &maps.a, &full, col, b * p.ctx_rows_a + qb * 64);
      ptx::tma_load_2d(base + (2 + c) * BST_TILE, &maps.b, &full, col, b * p.ctx_rows_b + kb * 64);
    }
  }
  __syncthreads();
  float acc[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) acc[i] = 0.f;
  if (!ptx::mbar_wait(&full, 0)) g_tc_error = 21;
  ptx::wg_fence();
  for (int c = 0; c < chunks; ++c)
#pragma unroll
    for (int ks = 0; ks < 4; ++ks)
      ptx::wgmma_n64<BF16, 0, 0>(acc, ptx::make_desc(base + c * BST_TILE + ks * 32, 16, 1024, ptx::SWZ_128B),
                                 ptx::make_desc(base + (2 + c) * BST_TILE + ks * 32, 16, 1024, ptx::SWZ_128B));
  ptx::wg_commit();
  ptx::wg_wait<0>();
  ptx::wg_fence_regs(acc);

  TC* out = reinterpret_cast<TC*>(p.c) + ((size_t)z * p.blocks + blk) * 64 * 64;
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const int row = warp * 16 + lane / 4 + 8 * hh;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int col = 8 * j + 2 * (lane % 4);
      const float v0 = acc[4 * j + 2 * hh], v1 = acc[4 * j + 2 * hh + 1];
      if constexpr (sizeof(TC) == 4) *reinterpret_cast<float2*>(out + row * 64 + col) = make_float2(v0, v1);
      else *reinterpret_cast<uint32_t*>(out + row * 64 + col) = pack2<std::is_same<TC, __nv_bfloat16>::value>(v0, v1);
    }
  }
}

// ------------------------------------------------------------------------------------------------
struct BstXnParams {
  const int32_t* lut;       // [lut_heads][n_out + blocks][2]
  long long lut_head_stride;
  int n_out, heads, blocks, head_state;
  int ctx_rows_b, ctx_rows_c;
  void* c;
};
struct BstXnTmaps { CUtensorMap a, b; };

template <bool BF16, bool TRANS_A>
__global__ void __launch_bounds__(BST_THREADS)
tc_bst_xn_kernel(const BstXnParams p, const __grid_constant__ BstXnTmaps maps) {
  constexpr int ST = BST_STAGES;
  constexpr uint32_t STAGE_BYTES = 3 * BST_TILE;     // sparse block + up to two 64-column tiles of B (head_state <= 128)
  extern __shared__ uint8_t smem_raw[];
  __shared__ uint64_t full[ST];
  const uint32_t base = aligned_smem_base(smem_raw);
  const int tid = threadIdx.x, warp = tid / 32, lane = tid % 32;
  const int chunks = p.head_state / 64;
  const int o = (int)(blockIdx.x % (unsigned)p.n_out);
  const int z = (int)(blockIdx.x / (unsigned)p.n_out);
  const int b = z / p.heads, h = z % p.heads;
  const int32_t* lut = p.lut + h * p.lut_head_stride;
  const int first = lut[2 * o], count = lut[2 * o + 1];
  const int2* ent = reinterpret_cast<const int2*>(lut) + first;

  auto issue = [&](int e) {                          // one thread: stage entry e = (sparse block, input block)
    const int2 bi = ent[e];
    const uint32_t st = base + (uint32_t)(e % ST) * STAGE_BYTES;
    uint64_t* bar = &full[e % ST];
    ptx::mbar_expect_tx(bar, (uint32_t)(1 + chunks) * BST_TILE);
    ptx::tma_load_2d(st, &maps.a, bar, 0, (int)(((long long)z * p.blocks + bi.x) * 64));
    for (int c = 0; c < chunks; ++c)
      ptx::tma_load_2d(st + (1 + c) * BST_TILE, &maps.b, bar, h * p.head_state + c * 64, b * p.ctx_rows_b + bi.y * 64);
  };
  if (tid == 0) {
    for (int i = 0; i < ST; ++i) ptx::mbar_init(&full[i], 1);
    ptx::fence_mbar_init();
  }
  __syncthreads();
  if (tid == 0)
    for (int e = 0; e < count && e < ST; ++e) issue(e);

  float acc[2][32];
#pragma unroll
  for (int c = 0; c < 2; ++c)
#pragma unroll
    for (int i = 0; i < 32; ++i) acc[c][i] = 0.f;
  for (int e = 0; e < count; ++e) {
    const uint32_t st = base + (uint32_t)(e % ST) * STAGE_BYTES;
    if (!ptx::mbar_wait(&full[e % ST], (uint32_t)(e / ST) & 1)) g_tc_error = 31;
    ptx::wg_fence();
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
      // NN: A[i][j], M = i, K = j contiguous (K-major).  TN: A^T, M = j contiguous (MN-major), K=16 step = 16 rows.
      const uint64_t adesc = TRANS_A ? ptx::make_desc(st + ks * 2048, BST_TILE, 1024, ptx::SWZ_128B)
                                     : ptx::make_desc(st + ks * 32, 16, 1024, ptx::SWZ_128B);
      // B = dense tile [64 rows = K][64 columns = N], MN-major
      ptx::wgmma_n64<BF16, TRANS_A ? 1 : 0, 1>(acc[0], adesc, ptx::make_desc(st + BST_TILE + ks * 2048, BST_TILE, 1024, ptx::SWZ_128B));
      if (chunks == 2)
        ptx::wgmma_n64<BF16, TRANS_A ? 1 : 0, 1>(acc[1], adesc, ptx::make_desc(st + 2 * BST_TILE + ks * 2048, BST_TILE, 1024, ptx::SWZ_128B));
    }
    ptx::wg_commit();
    ptx::wg_wait<1>();
    __syncthreads();
    if (tid == 0 && e >= 1 && e - 1 + ST < count) issue(e - 1 + ST);
  }
  ptx::wg_wait<0>();
  ptx::wg_fence_regs(acc[0]);
  ptx::wg_fence_regs(acc[1]);

  // epilogue (also zero-fills output blocks whose LUT row is empty)
  const long long S = (long long)p.heads * p.head_state;
  uint16_t* cbase = reinterpret_cast<uint16_t*>(p.c);
  for (int c = 0; c < chunks; ++c)
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int row = warp * 16 + lane / 4 + 8 * hh;
      uint16_t* out = cbase + ((long long)b * p.ctx_rows_c + o * 64 + row) * S + (long long)h * p.head_state + c * 64;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int col = 8 * j + 2 * (lane % 4);
        const float v0 = c ? acc[1][4 * j + 2 * hh] : acc[0][4 * j + 2 * hh];
        const float v1 = c ? acc[1][4 * j + 2 * hh + 1] : acc[0][4 * j + 2 * hh + 1];
        *reinterpret_cast<uint32_t*>(out + col) = pack2<BF16>(v0, v1);
      }
    }
}

// ------------------------------------------------------------------------------------------------
inline bool bst_tc_applicable(int dtype, int bsize, int head_state, const void* a, const void* b, const void* c) {
  if (dtype != BSMM_F16 && dtype != BSMM_BF16) { fail(0, "fp32 runs on the FMA path"); return false; }
  if (bsize != 64) { fail(0, "block size %d uses the CUDA-core path", bsize); return false; }
  if (head_state != 64 && head_state != 128) { fail(0, "head_state %d uses the CUDA-core path", head_state); return false; }
  if (((uintptr_t)a | (uintptr_t)b | (uintptr_t)c) & 15) { fail(0, "pointers must be 16-byte aligned for TMA"); return false; }
  return wgmma_device();
}

inline int tc_bst_nt(int dtype, int c_dtype, int bsize, const int32_t* nt_lut, int lut_heads, int blocks,
                     const void* a, const void* b, void* c, int batch, int heads, int head_state, int ctx_blks_a,
                     int ctx_blks_b, cudaStream_t s) {
  if (!bst_tc_applicable(dtype, bsize, head_state, a, b, c)) return TC_NOT_APPLICABLE;
  const uint64_t S = (uint64_t)heads * head_state;
  BstNtTmaps maps;
  if (int e = cached_tmap_2d(&maps.a, dtype, a, S, (uint64_t)batch * ctx_blks_a * 64, S, 64, 64, CU_TENSOR_MAP_SWIZZLE_128B)) return e;
  if (int e = cached_tmap_2d(&maps.b, dtype, b, S, (uint64_t)batch * ctx_blks_b * 64, S, 64, 64, CU_TENSOR_MAP_SWIZZLE_128B)) return e;
  BstNtParams p;
  p.lut = nt_lut; p.lut_head_stride = lut_heads > 1 ? 2LL * blocks : 0;
  p.heads = heads; p.blocks = blocks; p.head_state = head_state;
  p.ctx_rows_a = ctx_blks_a * 64; p.ctx_rows_b = ctx_blks_b * 64; p.c = c;
  const size_t smem = 4 * BST_TILE + SMEM_ALIGN_SLACK;
  const unsigned grid = (unsigned)((long long)batch * heads * blocks);     // < 2^20: the output has < 2^32 elements
  const bool bf = dtype == BSMM_BF16;
#define BSMM_LAUNCH_NT(BFV, TCV)                                                         \
  { auto kern = tc_bst_nt_kernel<BFV, TCV>;                                              \
    static thread_local uint64_t cfg = 0;                                                \
    if (int e = ensure_dyn_smem(kern, smem, cfg)) return e;                              \
    kern<<<grid, BST_THREADS, smem, s>>>(p, maps); }
  if (c_dtype == BSMM_F32) { if (bf) BSMM_LAUNCH_NT(true, float) else BSMM_LAUNCH_NT(false, float) }
  else if (c_dtype == BSMM_BF16) { if (bf) BSMM_LAUNCH_NT(true, __nv_bfloat16) else BSMM_LAUNCH_NT(false, __nv_bfloat16) }
  else { if (bf) BSMM_LAUNCH_NT(true, __half) else BSMM_LAUNCH_NT(false, __half) }
#undef BSMM_LAUNCH_NT
  return check_launch("wgmma_bst_nt");
}

inline int tc_bst_xn(int a_dtype, int dtype, int bsize, int transpose_a, const int32_t* lut, int lut_heads, int blocks,
                     const void* a, const void* b, void* c, int batch, int heads, int head_state,
                     int ctx_blks_b, int ctx_blks_c, cudaStream_t s) {
  if (a_dtype != dtype) { fail(0, "mixed sparse/dense dtypes use the CUDA-core path"); return TC_NOT_APPLICABLE; }
  if (!bst_tc_applicable(dtype, bsize, head_state, a, b, c)) return TC_NOT_APPLICABLE;
  if ((unsigned long long)batch * heads * blocks * 64 >= (1ull << 31)) { fail(0, "sparse tensor too large for one tensor map"); return TC_NOT_APPLICABLE; }
  const uint64_t S = (uint64_t)heads * head_state;
  BstXnTmaps maps;
  if (int e = cached_tmap_2d(&maps.a, dtype, a, 64, (uint64_t)batch * heads * blocks * 64, 64, 64, 64, CU_TENSOR_MAP_SWIZZLE_128B)) return e;
  if (int e = cached_tmap_2d(&maps.b, dtype, b, S, (uint64_t)batch * ctx_blks_b * 64, S, 64, 64, CU_TENSOR_MAP_SWIZZLE_128B)) return e;
  BstXnParams p;
  p.lut = lut; p.lut_head_stride = lut_heads > 1 ? 2LL * (ctx_blks_c + blocks) : 0; p.n_out = ctx_blks_c;
  p.heads = heads; p.blocks = blocks; p.head_state = head_state;
  p.ctx_rows_b = ctx_blks_b * 64; p.ctx_rows_c = ctx_blks_c * 64; p.c = c;
  const size_t smem = (size_t)BST_STAGES * 3 * BST_TILE + SMEM_ALIGN_SLACK;
  const unsigned grid = (unsigned)((long long)batch * heads * ctx_blks_c);
#define BSMM_LAUNCH_XN(BFV, TRV)                                                         \
  { auto kern = tc_bst_xn_kernel<BFV, TRV>;                                              \
    static thread_local uint64_t cfg = 0;                                                \
    if (int e = ensure_dyn_smem(kern, smem, cfg)) return e;                              \
    kern<<<grid, BST_THREADS, smem, s>>>(p, maps); }
  const bool bf = dtype == BSMM_BF16;
  if (transpose_a) { if (bf) BSMM_LAUNCH_XN(true, true) else BSMM_LAUNCH_XN(false, true) }
  else { if (bf) BSMM_LAUNCH_XN(true, false) else BSMM_LAUNCH_XN(false, false) }
#undef BSMM_LAUNCH_XN
  return check_launch(transpose_a ? "wgmma_bst_tn" : "wgmma_bst_nn");
}

}  // namespace bsmm
