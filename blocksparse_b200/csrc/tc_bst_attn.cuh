// Fused block-sparse attention on wgmma, block size 64, head_state 64 / 128, fp16 / bf16:
//   o[b, q-blk, h, :] = softmax_row(mask(scale * Q K^T)) V     over the key blocks of the query block's nn_lut row.
// Computes what bst_nt -> bst_softmax -> bst_xn(NN) compute, without writing the scores or the probabilities: no single
// reference launcher corresponds to it.
//
// One CTA (one warpgroup) per (query block, head, batch) owns the block's 64 query rows.  The Q tile is staged once; the
// CTA then walks its LUT row, entry e = (block id, key block), through a ring of TMA stages that each hold the key and
// the value tile of one entry.  Per entry:
//   S = Q K^T          wgmma, both operands K-major (as tc_bst_nt_kernel), fp32 in registers, never stored;
//   scale, mask        masked keys -> -FLT_MAX (as bst_softmax: a row that sees no key gets uniform weights);
//   online softmax     running row max m and sum l; O and l are rescaled when m grows;
//   O += P V           P converted to the input dtype in registers is the A operand (register-A wgmma: the fp32
//                      accumulator layout of 16 score columns is the A fragment layout), V the MN-major B operand
//                      (as tc_bst_xn_kernel).
// The stage of entry e is refilled with entry e + ST once O += P V of entry e has retired.  The epilogue divides by l
// and stores 16-bit rows; an empty LUT row is written as zeros.  Accumulation follows LUT order: results are
// deterministic.  With STATS the epilogue also stores every row's final running max m and full sum l, which the fused
// backward (tc_bst_attn_bwd.cuh) needs to recompute P = exp(s - m) / l; o is the same either way.
//
// With DROP, attention dropout on the normalised probabilities: o_i = sum_j Z_ij exp(s_ij - m_i) v_j / (keep_prob l_i),
// l the sum over every visible key (Z does not enter it; nor m and l as stored), Z_ij the keep bit of element
// e = (((b heads + h) blocks + block id) 64 + i) 64 + j of the (batch, heads, blocks, 64, 64) probabilities, drawn as
// bsmm_dropout_mask draws it from the device (seed, call) (philox.cuh).  Z is applied to the unnormalised P before it
// enters P V, and 1 / keep_prob is folded into the epilogue's 1 / l.  A thread holds 2 rows x 16 keys of an entry; one
// Philox block covers 4 consecutive keys of a row, which two neighbouring lanes share, so each lane draws the blocks of
// one of its rows and the pair trade the halves they need in one shuffle: 8 Philox blocks per thread and entry, drawn
// while S = Q K^T runs on the tensor cores.
//
// Grouped-query attention: with k and v of kv_heads heads ((batch, ctx_k, kv_heads*head_state), group = heads /
// kv_heads) the K and V tensor maps have rows of kv_heads*head_state and query head h stages the tiles of kv head
// h / group.  Q, o, the statistics, the mask and the dropout elements stay query head h's, and each row walks the same
// data in the same LUT order, so o is bit-identical to this kernel's on k and v expanded to heads heads.
#pragma once
#include <float.h>
#include "philox.cuh"
#include "softmax.cuh"
#include "tc_bst.cuh"

namespace bsmm {

constexpr int BST_ATTN_STAGES = 2;

struct BstAttnParams {
  const int32_t* lut;             // nn_lut: [lut_heads][ctx_blks_q + blocks][2]
  long long lut_head_stride;
  const uint64_t* mask;           // uint64 [mask_heads][blocks][64] or null
  long long mask_head_stride;     // words
  int autoregress_at_key;         // < 0: off
  float scale;
  int n_q, heads, head_state;     // n_q = ctx_blks_q
  int ctx_rows_q, ctx_rows_k;
  void* o;
  float* row_max;                 // STATS: [batch][heads][ctx_rows_q] final running max m and full sum l of each row
  float* row_sum;
  const long long* seed_call;     // DROP: device [seed, call], read only
  unsigned long long keep_thr;    // DROP: floor(keep_prob 2^32)
  float keep_prob, rkeep;         // DROP: keep_prob and fp32(1 / keep_prob)
  int blocks;                     // blocks of the layout (the element index of the dropout mask)
  int group;                      // query heads per key / value head: head h reads kv head h / group
};

// Keep bits of this thread's two rows r0 + 8hh (hh = 0, 1) and 16 keys of one entry: bit 4j + x of kw[hh] is key
// 8j + 2(lane%4) + x (accumulator layout, ptx.cuh).  rows0 = (b heads + h) blocks + block id, the entry's first row of
// the mask in 64-row units.
__device__ __forceinline__ void attn_keep_bits(uint32_t (&kw)[2], unsigned long long rows0, int r0, int lane,
                                               unsigned long long call, uint2 key, unsigned long long thr) {
  const int pp = lane & 1;                              // this lane draws row r0 + 8pp, its partner lane ^ 1 the other
  const unsigned long long g0 = (rows0 * 64 + r0 + 8 * pp) * 16 + ((lane % 4) >> 1);
  uint32_t mine = 0;
#pragma unroll
  for (int j = 0; j < 8; ++j) mine |= philox_keep4(g0 + 2 * j, call, key, thr) << (4 * j);
  const uint32_t other = __shfl_xor_sync(0xffffffffu, mine, 1);
  kw[0] = (pp == 0 ? mine : other) >> (2 * pp);         // this lane's keys are words 2pp, 2pp + 1 of each block
  kw[1] = (pp == 1 ? mine : other) >> (2 * pp);
}
struct BstAttnTmaps { CUtensorMap q, k, v; };

template <bool BF16, int CH, bool STATS = false, bool DROP = false>      // CH = head_state / 64
__global__ void __launch_bounds__(BST_THREADS)
wgmma_bst_attention(const BstAttnParams p, const __grid_constant__ BstAttnTmaps maps) {
  constexpr int ST = BST_ATTN_STAGES;
  constexpr uint32_t KV_BYTES = CH * BST_TILE;          // one key (or value) tile of one entry
  constexpr uint32_t STAGE_BYTES = 2 * KV_BYTES;        // key tile, then value tile
  constexpr float LOG2E = 1.4426950408889634f;
  extern __shared__ uint8_t smem_raw[];
  __shared__ uint64_t qbar, full[ST];
  const uint32_t base = aligned_smem_base(smem_raw);    // Q chunks, then the ring
  const uint32_t ring = base + KV_BYTES;
  const int tid = threadIdx.x, warp = tid / 32, lane = tid % 32;
  const int qb = (int)(blockIdx.x % (unsigned)p.n_q);
  const int z = (int)(blockIdx.x / (unsigned)p.n_q);
  const int b = z / p.heads, h = z % p.heads;
  const int32_t* lut = p.lut + h * p.lut_head_stride;
  const int first = lut[2 * qb], count = lut[2 * qb + 1];
  const int2* ent = reinterpret_cast<const int2*>(lut) + first;
  const int col0 = h * p.head_state;
  const int kcol0 = (h / p.group) * p.head_state;       // K and V: the columns of kv head h / group

  auto issue = [&](int e) {                             // one thread: stage entry e = (block id, key block)
    const int kb = ent[e].y;
    const uint32_t st = ring + (uint32_t)(e % ST) * STAGE_BYTES;
    uint64_t* bar = &full[e % ST];
    ptx::mbar_expect_tx(bar, STAGE_BYTES);
    for (int c = 0; c < CH; ++c) {
      ptx::tma_load_2d(st + c * BST_TILE, &maps.k, bar, kcol0 + c * 64, b * p.ctx_rows_k + kb * 64);
      ptx::tma_load_2d(st + KV_BYTES + c * BST_TILE, &maps.v, bar, kcol0 + c * 64, b * p.ctx_rows_k + kb * 64);
    }
  };
  if (tid == 0) {
    ptx::mbar_init(&qbar, 1);
    for (int i = 0; i < ST; ++i) ptx::mbar_init(&full[i], 1);
    ptx::fence_mbar_init();
  }
  __syncthreads();
  if (tid == 0 && count > 0) {
    ptx::mbar_expect_tx(&qbar, KV_BYTES);
    for (int c = 0; c < CH; ++c)
      ptx::tma_load_2d(base + c * BST_TILE, &maps.q, &qbar, col0 + c * 64, b * p.ctx_rows_q + qb * 64);
    for (int e = 0; e < count && e < ST; ++e) issue(e);
  }

  // This thread's two query rows (accumulator layout, ptx.cuh): r0 = 16 warp + lane/4 and r0 + 8.
  const int r0 = warp * 16 + lane / 4;
  const uint64_t* mask = p.mask ? p.mask + (p.mask_head_stride ? h * p.mask_head_stride : 0) : nullptr;
  float o[CH][32];
#pragma unroll
  for (int c = 0; c < CH; ++c)
#pragma unroll
    for (int i = 0; i < 32; ++i) o[c][i] = 0.f;
  float m[2] = {-FLT_MAX, -FLT_MAX}, l[2] = {0.f, 0.f};   // l: this thread's part of the row sum
  uint2 key = make_uint2(0u, 0u);
  unsigned long long call = 0;
  if constexpr (DROP) {
    const unsigned long long seed = (unsigned long long)p.seed_call[0];
    call = (unsigned long long)p.seed_call[1];
    key = make_uint2((unsigned)seed, (unsigned)(seed >> 32));
  }
  if (count > 0 && !ptx::mbar_wait(&qbar, 0)) g_tc_error = 41;

  for (int e = 0; e < count; ++e) {
    const uint32_t st = ring + (uint32_t)(e % ST) * STAGE_BYTES;
    if (!ptx::mbar_wait(&full[e % ST], (uint32_t)(e / ST) & 1)) g_tc_error = 42;
    float s[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) s[i] = 0.f;
    ptx::wg_fence();
#pragma unroll
    for (int c = 0; c < CH; ++c)
#pragma unroll
      for (int ks = 0; ks < 4; ++ks)
        ptx::wgmma_n64<BF16, 0, 0>(s, ptx::make_desc(base + c * BST_TILE + ks * 32, 16, 1024, ptx::SWZ_128B),
                                   ptx::make_desc(st + c * BST_TILE + ks * 32, 16, 1024, ptx::SWZ_128B));
    ptx::wg_commit();
    uint32_t kw[2];                                     // the entry's keep bits, drawn while the MMAs run
    if constexpr (DROP)
      attn_keep_bits(kw, ((unsigned long long)b * p.heads + h) * p.blocks + ent[e].x, r0, lane, call, key, p.keep_thr);
    ptx::wg_wait<0>();
    ptx::wg_fence_regs(s);

    // scale, then mask (the order of bst_softmax); s[4j + 2hh + x] is key 8j + 2(lane%4) + x of row r0 + 8hh
    const int2 bk = ent[e];
#pragma unroll
    for (int i = 0; i < 32; ++i) s[i] *= p.scale;
    if (mask) {
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        uint64_t w = mask[(long long)bk.x * 64 + r0 + 8 * hh];
        if (p.autoregress_at_key >= 0) w = autoregress_word<64>(w, p.autoregress_at_key, bk.y, qb * 64 + r0 + 8 * hh);
        if (w != ~0ull) {
          const uint64_t mine = w >> (2 * (lane % 4));
#pragma unroll
          for (int j = 0; j < 8; ++j)
#pragma unroll
            for (int x = 0; x < 2; ++x)
              if (!((mine >> (8 * j + x)) & 1ull)) s[4 * j + 2 * hh + x] = -FLT_MAX;
        }
      }
    }

    // online softmax: the 4 lanes of a quad share a row
    float alpha[2];
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      float mx = m[hh];
#pragma unroll
      for (int j = 0; j < 8; ++j) mx = fmaxf(mx, fmaxf(s[4 * j + 2 * hh], s[4 * j + 2 * hh + 1]));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      alpha[hh] = exp2f((m[hh] - mx) * LOG2E);          // subtract first: -FLT_MAX * LOG2E overflows
      m[hh] = mx;
      float acc = 0.f;
#pragma unroll
      for (int j = 0; j < 8; ++j)
#pragma unroll
        for (int x = 0; x < 2; ++x) {
          float& v = s[4 * j + 2 * hh + x];
          v = exp2f((v - mx) * LOG2E);
          acc += v;
          if constexpr (DROP) if (!((kw[hh] >> (4 * j + x)) & 1u)) v = 0.f;   // after the row sum: l is not affected
        }
      l[hh] = l[hh] * alpha[hh] + acc;
    }
#pragma unroll
    for (int c = 0; c < CH; ++c)
#pragma unroll
      for (int i = 0; i < 32; ++i) o[c][i] *= alpha[(i >> 1) & 1];

    // P in the input dtype, as the A fragments of the four K = 16 slices
    uint32_t a[4][4];
#pragma unroll
    for (int kk = 0; kk < 4; ++kk)
#pragma unroll
      for (int r = 0; r < 4; ++r) a[kk][r] = pack2<BF16>(s[8 * kk + 2 * r], s[8 * kk + 2 * r + 1]);
    ptx::wg_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk)
#pragma unroll
      for (int c = 0; c < CH; ++c)   // V = [64 keys = K][64 state columns = N], MN-major
        ptx::wgmma_rs_n64<BF16, 1>(o[c], a[kk], ptx::make_desc(st + KV_BYTES + c * BST_TILE + kk * 2048, BST_TILE, 1024, ptx::SWZ_128B));
    ptx::wg_commit();
    ptx::wg_wait<0>();
#pragma unroll
    for (int c = 0; c < CH; ++c) ptx::wg_fence_regs(o[c]);
    __syncthreads();                                    // every warp's MMAs that read this stage have retired
    if (tid == 0 && e + ST < count) issue(e + ST);
  }

  // epilogue: full row sums, normalise, store (an empty LUT row leaves o = 0 and writes zeros)
  const long long S = (long long)p.heads * p.head_state;
  uint16_t* obase = reinterpret_cast<uint16_t*>(p.o);
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    float sum = l[hh];
    sum += __shfl_xor_sync(0xffffffffu, sum, 1);
    sum += __shfl_xor_sync(0xffffffffu, sum, 2);
    float inv;
    if constexpr (DROP) inv = count > 0 ? p.rkeep / sum : 0.f;
    else inv = count > 0 ? 1.f / sum : 0.f;
    const int row = r0 + 8 * hh;
    if (STATS && lane % 4 == 0) {                       // m is already the quad's common value
      const long long r = ((long long)b * p.heads + h) * p.ctx_rows_q + qb * 64 + row;
      p.row_max[r] = m[hh];
      p.row_sum[r] = sum;
    }
    uint16_t* out = obase + ((long long)b * p.ctx_rows_q + qb * 64 + row) * S + col0;
#pragma unroll
    for (int c = 0; c < CH; ++c)
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int col = c * 64 + 8 * j + 2 * (lane % 4);
        *reinterpret_cast<uint32_t*>(out + col) = pack2<BF16>(o[c][4 * j + 2 * hh] * inv, o[c][4 * j + 2 * hh + 1] * inv);
      }
  }
}

// ------------------------------------------------------------------------------------------------
// Dropout of the fused kernels: keep_prob in (0, 1), seed_call the device [seed, call] (never written).  A null
// BstAttnDrop runs the kernels without dropout.
struct BstAttnDrop {
  double keep_prob;
  const long long* seed_call;
};

template <typename P> inline void set_drop(P& p, const BstAttnDrop* drop) {
  p.seed_call = drop ? drop->seed_call : nullptr;
  p.keep_thr = drop ? (unsigned long long)floor(drop->keep_prob * 4294967296.0) : 0;   // as bsmm_dropout_mask
  p.keep_prob = drop ? (float)drop->keep_prob : 1.f;
  p.rkeep = drop ? (float)(1.0 / drop->keep_prob) : 1.f;                              // as bsmm_dropout_apply
}

inline int tc_bst_attention(int dtype, int bsize, const int32_t* nn_lut, int lut_heads, int blocks, const void* mask,
                            int mask_heads, int autoregress_at_key, const void* q, const void* k, const void* v, void* o,
                            float scale, int batch, int heads, int head_state, int ctx_blks_q, int ctx_blks_k,
                            cudaStream_t s, float* row_max = nullptr, float* row_sum = nullptr,
                            const BstAttnDrop* drop = nullptr, int kv_heads = 0) {
  if ((uintptr_t)o & 15) { fail(0, "pointers must be 16-byte aligned for TMA"); return TC_NOT_APPLICABLE; }
  if (!bst_tc_applicable(dtype, bsize, head_state, q, k, v)) return TC_NOT_APPLICABLE;
  if (kv_heads <= 0) kv_heads = heads;                  // k and v are (batch, ctx_k, kv_heads * head_state)
  const uint64_t S = (uint64_t)heads * head_state, SKV = (uint64_t)kv_heads * head_state;
  BstAttnTmaps maps;
  if (int e = cached_tmap_2d(&maps.q, dtype, q, S, (uint64_t)batch * ctx_blks_q * 64, S, 64, 64, CU_TENSOR_MAP_SWIZZLE_128B)) return e;
  if (int e = cached_tmap_2d(&maps.k, dtype, k, SKV, (uint64_t)batch * ctx_blks_k * 64, SKV, 64, 64, CU_TENSOR_MAP_SWIZZLE_128B)) return e;
  if (int e = cached_tmap_2d(&maps.v, dtype, v, SKV, (uint64_t)batch * ctx_blks_k * 64, SKV, 64, 64, CU_TENSOR_MAP_SWIZZLE_128B)) return e;
  BstAttnParams p;
  p.lut = nn_lut; p.lut_head_stride = lut_heads > 1 ? 2LL * (ctx_blks_q + blocks) : 0;
  p.mask = reinterpret_cast<const uint64_t*>(mask);
  p.mask_head_stride = (mask && mask_heads > 1) ? (long long)blocks * 64 : 0;
  p.autoregress_at_key = autoregress_at_key; p.scale = scale;
  p.n_q = ctx_blks_q; p.heads = heads; p.head_state = head_state;
  p.ctx_rows_q = ctx_blks_q * 64; p.ctx_rows_k = ctx_blks_k * 64; p.o = o;
  p.row_max = row_max; p.row_sum = row_sum;
  set_drop(p, drop);
  p.blocks = blocks;
  p.group = heads / kv_heads;
  const bool stats = row_max != nullptr;
  const int ch = head_state / 64;
  const size_t smem = (size_t)(1 + 2 * BST_ATTN_STAGES) * ch * BST_TILE + SMEM_ALIGN_SLACK;
  const unsigned grid = (unsigned)((long long)batch * heads * ctx_blks_q);
#define BSMM_LAUNCH_ATTN(BFV, CHV, STV, DRV)                                             \
  { auto kern = wgmma_bst_attention<BFV, CHV, STV, DRV>;                                 \
    static thread_local uint64_t cfg = 0;                                                \
    if (int e = ensure_dyn_smem(kern, smem, cfg)) return e;                              \
    kern<<<grid, BST_THREADS, smem, s>>>(p, maps); }
#define BSMM_LAUNCH_ATTN_CH(BFV, STV, DRV) \
  { if (ch == 2) BSMM_LAUNCH_ATTN(BFV, 2, STV, DRV) else BSMM_LAUNCH_ATTN(BFV, 1, STV, DRV) }
#define BSMM_LAUNCH_ATTN_BF(STV, DRV) \
  { if (bf) BSMM_LAUNCH_ATTN_CH(true, STV, DRV) else BSMM_LAUNCH_ATTN_CH(false, STV, DRV) }
  const bool bf = dtype == BSMM_BF16;
  if (drop) { if (stats) BSMM_LAUNCH_ATTN_BF(true, true) else BSMM_LAUNCH_ATTN_BF(false, true) }
  else { if (stats) BSMM_LAUNCH_ATTN_BF(true, false) else BSMM_LAUNCH_ATTN_BF(false, false) }
#undef BSMM_LAUNCH_ATTN_BF
#undef BSMM_LAUNCH_ATTN_CH
#undef BSMM_LAUNCH_ATTN
  if (drop) return check_launch(stats ? "wgmma_bst_attention_train_dropout" : "wgmma_bst_attention_dropout");
  return check_launch(stats ? "wgmma_bst_attention_train" : "wgmma_bst_attention");
}

}  // namespace bsmm
