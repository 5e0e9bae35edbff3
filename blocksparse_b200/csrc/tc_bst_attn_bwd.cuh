// Fused backward of block-sparse attention on wgmma, block size 64, head_state 64 / 128, fp16 / bf16.  With
// P = softmax_row(mask(scale * Q K^T)) and O = P V (tc_bst_attn.cuh), and dO the gradient of O:
//   dV = P^T dO,   dP = dO V^T,   D_i = sum_c dO[i,c] O[i,c],   dS = scale * P o (dP - D),   dQ = dS K,   dK = dS^T Q
// over the blocks of the layout.  D is the row sum of dP o P that bst_softmax_grad forms (sum_j dP_ij P_ij = dO_i . O_i).
// P is recomputed from the scores and the forward's row statistics, P = exp(s - m) / l, so neither the scores, the
// probabilities nor dS are ever written.  Computes what the chain's backward (bst_nt, bst_softmax, bst_xn TN,
// bst_nt, bst_softmax_grad, bst_xn TN and NN) computes; no single reference launcher corresponds to it.
//
// Two kernels, run in this order on one stream:
//   wgmma_bst_attention_bwd_dq    one warpgroup per (query block, head, batch).  Prologue: D of its 64 rows in fp32
//                                 from the saved 16-bit o, stored to a [batch][heads][ctx_q] workspace.  Then it walks
//                                 the block's nn_lut row through a ring of TMA stages holding the key and value tiles
//                                 of one entry (Q and dO are staged once):
//                                   S = Q K^T, dP = dO V^T   both operands K-major;
//                                   P, dS                    scale and mask as the forward, then the formulas above;
//                                   dQ += dS K               dS in the input dtype as the register A operand, K MN-major.
//   wgmma_bst_attention_bwd_dkdv  one CTA per (key block, head, batch), launched longest tn_lut row first (tn_order).
//                                 K and V are staged once; the CTA walks the key block's tn_lut row, entries (block id,
//                                 query block), through a ring of Q and dO tiles, with that query block's m, l and D:
//                                   S^T = K Q^T, dP^T = V dO^T; P^T; dV += P^T dO; dS^T; dK += dS^T Q.
//                                 Here a thread holds key rows and query columns: the mask bit of (query j, key i) is bit
//                                 i of word j of the block, so each entry's 64 words (autoregress rewrite applied), m,
//                                 1/l and D are staged in shared memory.  At head_state 128 the CTA has two warpgroups:
//                                 both compute S^T and dP^T over the whole head_state, each owns 64 state columns of dK
//                                 and dV (one warpgroup holding all of both would need more than 255 registers).
// Grouped-query attention (kv_heads < heads, group g = heads / kv_heads, query head h reading kv head h / g): the dq
// kernel stages kv head h / g's tiles and is otherwise unchanged.  The dkdv kernel runs one CTA per (key block, kv head,
// batch), launched in the order of the group's first head; it stages K and V once and walks the tn_lut rows of the
// group's heads h = kvh g + j, j ascending, each in LUT order, through the same ring, with head h's mask, m, l, D and
// keep bits, so dK and dV sum the whole group in fp32 registers and are rounded once.  g = 1 is the kernel above.
// An empty LUT row writes zeros (dQ of a query block no key is listed for, dK / dV of a key block no query sees).  No
// atomics; accumulation follows LUT order: results are deterministic.  A row whose keys are all masked has m = -FLT_MAX
// and uniform P = 1 / l; as in the chain, its dS = scale * P o (dP - D) reaches dQ and dK.
//
// With DROP, the backward of attention dropout (tc_bst_attn.cuh) with the forward's keep bits Z, regenerated from the
// same device (seed, call): dV = (P o Z)^T dO / keep_prob, dP = (dO V^T) o Z / keep_prob, D as above (dO . O),
// dS = scale P o (dP - D), computed as (scale / keep_prob) P o (Z o dO V^T - keep_prob D) so that 1 / keep_prob costs
// no multiply per element (the staged D is multiplied by keep_prob once per row, dV by 1 / keep_prob in the epilogue).
// The dq kernel draws the bits of its rows as the forward does; the dkdv kernel, whose threads hold key rows, draws
// each entry's 64 x 64 bits cooperatively into 64 shared words laid out as its mask words (bit key of word query).
// Both draw while the entry's S and dP MMAs run.
#pragma once
#include <float.h>
#include "tc_bst_attn.cuh"

namespace bsmm {

constexpr int BST_BWD_STAGES = 2;

struct BstAttnBwdParams {
  const int32_t* nn_lut;          // [lut_heads][ctx_blks_q + blocks][2]
  const int32_t* tn_lut;          // [lut_heads][ctx_blks_k + blocks][2]
  const int32_t* tn_order;        // [lut_heads][ctx_blks_k]: key blocks, longest tn_lut row first
  long long nn_head_stride, tn_head_stride, order_head_stride;
  const uint64_t* mask;           // uint64 [mask_heads][blocks][64] or null
  long long mask_head_stride;     // words
  int autoregress_at_key;         // < 0: off
  float scale;
  int n_q, n_k, batch, heads, head_state;
  int ctx_rows_q, ctx_rows_k;
  const void* o;                  // forward output, (batch, ctx_q, heads*head_state)
  const void* dy;                 // its gradient, same layout
  const float* row_max;           // [batch][heads][ctx_rows_q], from bst_attention_train
  const float* row_sum;
  float* delta;                   // [batch][heads][ctx_rows_q]: written by the dq kernel, read by the dkdv kernel
  void *dq, *dk, *dv;
  const long long* seed_call;     // DROP: as BstAttnParams
  unsigned long long keep_thr;
  float keep_prob, rkeep;
  int blocks;
  int kv_heads, group;            // k, v, dk, dv: (batch, ctx_k, kv_heads*head_state); head h reads kv head h / group
};
struct BstAttnBwdTmaps { CUtensorMap q, k, v, dy; };

// The eight 16-bit elements of one 16-byte vector as float.
template <bool BF16> __device__ __forceinline__ void unpack8(const uint4& u, float (&f)[8]) {
  const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    if constexpr (BF16) {
      const __nv_bfloat162 h = *reinterpret_cast<const __nv_bfloat162*>(&w[i]);
      f[2 * i] = __low2float(h); f[2 * i + 1] = __high2float(h);
    } else {
      const __half2 h = *reinterpret_cast<const __half2*>(&w[i]);
      f[2 * i] = __low2float(h); f[2 * i + 1] = __high2float(h);
    }
  }
}

// Stores a 64-row accumulator chunk (accumulator layout, ptx.cuh) as 16-bit rows of `out` (row pitch S elements).
template <bool BF16> __device__ __forceinline__ void store_rows(uint16_t* out, long long S, int r0, int lane,
                                                                const float (&acc)[32]) {
#pragma unroll
  for (int hh = 0; hh < 2; ++hh)
#pragma unroll
    for (int j = 0; j < 8; ++j)
      *reinterpret_cast<uint32_t*>(out + (r0 + 8 * hh) * S + 8 * j + 2 * (lane % 4)) =
          pack2<BF16>(acc[4 * j + 2 * hh], acc[4 * j + 2 * hh + 1]);
}

// ------------------------------------------------------------------------------------------------
template <bool BF16, int CH, bool DROP = false>      // CH = head_state / 64
__global__ void __launch_bounds__(BST_THREADS)
wgmma_bst_attention_bwd_dq(const BstAttnBwdParams p, const __grid_constant__ BstAttnBwdTmaps maps) {
  constexpr int ST = BST_BWD_STAGES;
  constexpr uint32_t T_BYTES = CH * BST_TILE;           // one 64-row tile of one operand, head_state columns
  constexpr uint32_t STAGE_BYTES = 2 * T_BYTES;         // key tile, then value tile
  constexpr float LOG2E = 1.4426950408889634f;
  extern __shared__ uint8_t smem_raw[];
  __shared__ uint64_t qbar, full[ST];
  __shared__ float s_delta[64];
  const uint32_t base = aligned_smem_base(smem_raw);    // Q, dO, then the ring
  const uint32_t dob = base + T_BYTES, ring = base + 2 * T_BYTES;
  const int tid = threadIdx.x, warp = tid / 32, lane = tid % 32;
  const int qb = (int)(blockIdx.x % (unsigned)p.n_q);
  const int z = (int)(blockIdx.x / (unsigned)p.n_q);
  const int b = z / p.heads, h = z % p.heads;
  const int32_t* lut = p.nn_lut + h * p.nn_head_stride;
  const int first = lut[2 * qb], count = lut[2 * qb + 1];
  const int2* ent = reinterpret_cast<const int2*>(lut) + first;
  const int col0 = h * p.head_state;
  const int kcol0 = (h / p.group) * p.head_state;       // K and V: the columns of kv head h / group
  const long long S = (long long)p.heads * p.head_state;
  const long long row0 = (long long)b * p.ctx_rows_q + qb * 64;            // first dense row of the block
  const long long stat0 = ((long long)b * p.heads + h) * p.ctx_rows_q + qb * 64;

  auto issue = [&](int e) {                             // one thread: stage entry e = (block id, key block)
    const int kb = ent[e].y;
    const uint32_t st = ring + (uint32_t)(e % ST) * STAGE_BYTES;
    uint64_t* bar = &full[e % ST];
    ptx::mbar_expect_tx(bar, STAGE_BYTES);
    for (int c = 0; c < CH; ++c) {
      ptx::tma_load_2d(st + c * BST_TILE, &maps.k, bar, kcol0 + c * 64, b * p.ctx_rows_k + kb * 64);
      ptx::tma_load_2d(st + T_BYTES + c * BST_TILE, &maps.v, bar, kcol0 + c * 64, b * p.ctx_rows_k + kb * 64);
    }
  };
  if (tid == 0) {
    ptx::mbar_init(&qbar, 1);
    for (int i = 0; i < ST; ++i) ptx::mbar_init(&full[i], 1);
    ptx::fence_mbar_init();
  }
  __syncthreads();
  if (tid == 0 && count > 0) {
    ptx::mbar_expect_tx(&qbar, 2 * T_BYTES);
    for (int c = 0; c < CH; ++c) {
      ptx::tma_load_2d(base + c * BST_TILE, &maps.q, &qbar, col0 + c * 64, (int)row0);
      ptx::tma_load_2d(dob + c * BST_TILE, &maps.dy, &qbar, col0 + c * 64, (int)row0);
    }
    for (int e = 0; e < count && e < ST; ++e) issue(e);
  }

  {  // D = rowsum(dO o O) in fp32: two threads per row, each half of the head's columns, in column order
    const int row = tid / 2, half = tid % 2;
    constexpr int HALF = CH * 32;                       // columns per thread
    const uint16_t* orow = reinterpret_cast<const uint16_t*>(p.o) + (row0 + row) * S + col0 + half * HALF;
    const uint16_t* drow = reinterpret_cast<const uint16_t*>(p.dy) + (row0 + row) * S + col0 + half * HALF;
    float acc = 0.f;
#pragma unroll
    for (int v = 0; v < HALF / 8; ++v) {
      float fo[8], fd[8];
      unpack8<BF16>(*reinterpret_cast<const uint4*>(orow + 8 * v), fo);
      unpack8<BF16>(*reinterpret_cast<const uint4*>(drow + 8 * v), fd);
#pragma unroll
      for (int i = 0; i < 8; ++i) acc = fmaf(fd[i], fo[i], acc);
    }
    acc += __shfl_xor_sync(0xffffffffu, acc, 1);
    if (half == 0) {
      s_delta[row] = acc;
      p.delta[stat0 + row] = acc;
    }
  }
  __syncthreads();

  // This thread's two query rows (accumulator layout, ptx.cuh): r0 = 16 warp + lane/4 and r0 + 8.
  const int r0 = warp * 16 + lane / 4;
  const uint64_t* mask = p.mask ? p.mask + (p.mask_head_stride ? h * p.mask_head_stride : 0) : nullptr;
  float m[2], il[2], dd[2];
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    m[hh] = p.row_max[stat0 + r0 + 8 * hh];
    il[hh] = count > 0 ? 1.f / p.row_sum[stat0 + r0 + 8 * hh] : 0.f;
    dd[hh] = s_delta[r0 + 8 * hh];
    if constexpr (DROP) dd[hh] *= p.keep_prob;
  }
  uint2 key = make_uint2(0u, 0u);
  unsigned long long call = 0;
  if constexpr (DROP) {
    const unsigned long long seed = (unsigned long long)p.seed_call[0];
    call = (unsigned long long)p.seed_call[1];
    key = make_uint2((unsigned)seed, (unsigned)(seed >> 32));
  }
  float dq[CH][32];
#pragma unroll
  for (int c = 0; c < CH; ++c)
#pragma unroll
    for (int i = 0; i < 32; ++i) dq[c][i] = 0.f;
  if (count > 0 && !ptx::mbar_wait(&qbar, 0)) g_tc_error = 51;

  for (int e = 0; e < count; ++e) {
    const uint32_t st = ring + (uint32_t)(e % ST) * STAGE_BYTES;
    if (!ptx::mbar_wait(&full[e % ST], (uint32_t)(e / ST) & 1)) g_tc_error = 52;
    float s[32], dp[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) { s[i] = 0.f; dp[i] = 0.f; }
    ptx::wg_fence();
#pragma unroll
    for (int c = 0; c < CH; ++c)
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
        ptx::wgmma_n64<BF16, 0, 0>(s, ptx::make_desc(base + c * BST_TILE + ks * 32, 16, 1024, ptx::SWZ_128B),
                                   ptx::make_desc(st + c * BST_TILE + ks * 32, 16, 1024, ptx::SWZ_128B));
        ptx::wgmma_n64<BF16, 0, 0>(dp, ptx::make_desc(dob + c * BST_TILE + ks * 32, 16, 1024, ptx::SWZ_128B),
                                   ptx::make_desc(st + T_BYTES + c * BST_TILE + ks * 32, 16, 1024, ptx::SWZ_128B));
      }
    ptx::wg_commit();
    uint32_t kw[2];                                     // the entry's keep bits, drawn while the MMAs run
    if constexpr (DROP)
      attn_keep_bits(kw, ((unsigned long long)b * p.heads + h) * p.blocks + ent[e].x, r0, lane, call, key, p.keep_thr);
    ptx::wg_wait<0>();
    ptx::wg_fence_regs(s);
    ptx::wg_fence_regs(dp);

    // scale, then mask (as the forward); s[4j + 2hh + x] is key 8j + 2(lane%4) + x of row r0 + 8hh
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
    // P = exp(s - m) / l, dS = scale P (dP - D), as the A fragments of the four K = 16 slices
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      const int hh = (i >> 1) & 1;
      const float pr = exp2f((s[i] - m[hh]) * LOG2E) * il[hh];   // subtract first: -FLT_MAX * LOG2E overflows
      if constexpr (DROP) {                             // dd = keep_prob D
        const float dpz = (kw[hh] >> (4 * (i >> 2) + (i & 1))) & 1u ? dp[i] : 0.f;
        s[i] = (p.scale * p.rkeep) * (pr * (dpz - dd[hh]));
      } else {
        s[i] = p.scale * (pr * (dp[i] - dd[hh]));
      }
    }
    uint32_t a[4][4];
#pragma unroll
    for (int kk = 0; kk < 4; ++kk)
#pragma unroll
      for (int r = 0; r < 4; ++r) a[kk][r] = pack2<BF16>(s[8 * kk + 2 * r], s[8 * kk + 2 * r + 1]);
    ptx::wg_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk)
#pragma unroll
      for (int c = 0; c < CH; ++c)   // K = [64 keys = K][64 state columns = N], MN-major
        ptx::wgmma_rs_n64<BF16, 1>(dq[c], a[kk], ptx::make_desc(st + c * BST_TILE + kk * 2048, BST_TILE, 1024, ptx::SWZ_128B));
    ptx::wg_commit();
    ptx::wg_wait<0>();
#pragma unroll
    for (int c = 0; c < CH; ++c) ptx::wg_fence_regs(dq[c]);
    __syncthreads();                                    // every warp's MMAs that read this stage have retired
    if (tid == 0 && e + ST < count) issue(e + ST);
  }

  // epilogue (an empty LUT row leaves dq = 0 and writes zeros)
  uint16_t* out = reinterpret_cast<uint16_t*>(p.dq) + row0 * S + col0;
#pragma unroll
  for (int c = 0; c < CH; ++c) store_rows<BF16>(out + c * 64, S, r0, lane, dq[c]);
}

// ------------------------------------------------------------------------------------------------
template <bool BF16, int CH, bool DROP = false>   // CH = head_state / 64 = warpgroups; warpgroup g owns state columns [64g, 64g + 64)
__global__ void __launch_bounds__(BST_THREADS * CH)
wgmma_bst_attention_bwd_dkdv(const BstAttnBwdParams p, const __grid_constant__ BstAttnBwdTmaps maps) {
  constexpr int ST = BST_BWD_STAGES;
  constexpr uint32_t T_BYTES = CH * BST_TILE;
  constexpr uint32_t STAGE_BYTES = 2 * T_BYTES;         // query tile, then dO tile
  constexpr float LOG2E = 1.4426950408889634f;
  extern __shared__ uint8_t smem_raw[];
  __shared__ uint64_t kvbar, full[ST];
  __shared__ uint64_t s_mask[64];
  __shared__ float s_m[64], s_il[64], s_d[64];
  __shared__ uint64_t s_keep[DROP ? 64 : 1];           // DROP: keep bit of (query j, key i) = bit i of word j
  const uint32_t base = aligned_smem_base(smem_raw);    // K, V, then the ring
  const uint32_t vb = base + T_BYTES, ring = base + 2 * T_BYTES;
  const int tid = threadIdx.x, wg = tid / BST_THREADS, warp = (tid % BST_THREADS) / 32, lane = tid % 32;
  const int Z = p.batch * p.kv_heads;
  const int i = (int)(blockIdx.x / (unsigned)Z);        // rank in the order of the group's first head
  const int z = (int)(blockIdx.x % (unsigned)Z);
  const int b = z / p.kv_heads, kvh = z % p.kv_heads;
  const int h0 = kvh * p.group;                         // the group's query heads are h0 .. h0 + group - 1
  const int kb = p.tn_order[h0 * p.order_head_stride + i];
  const int col0 = kvh * p.head_state;
  const long long S = (long long)p.heads * p.head_state, SKV = (long long)p.kv_heads * p.head_state;
  const long long krow0 = (long long)b * p.ctx_rows_k + kb * 64;
  // The CTA walks the key block's tn_lut rows of heads h0, h0 + 1, ... in turn, each in LUT order: entry (j, e) is
  // entry e of head h0 + j's row.  A cursor (j, e) steps through them; flat position f = entries before it.
  auto row_of = [&](int j, int& first) {                // count (and first entry) of head h0 + j's row
    const int32_t* lut = p.tn_lut + (long long)(h0 + j) * p.tn_head_stride;
    first = lut[2 * kb];
    return lut[2 * kb + 1];
  };
  int total = 0;
  for (int j = 0; j < p.group; ++j) { int f; total += row_of(j, f); }
  struct Cursor { int j, e, first, count; };
  auto start = [&](Cursor& c) {                         // the first entry
    c.j = 0; c.e = 0; c.count = row_of(0, c.first);
    while (c.count == 0 && c.j + 1 < p.group) c.count = row_of(++c.j, c.first);
  };
  auto step = [&](Cursor& c) {                          // the next entry, skipping heads whose row is empty
    if (++c.e < c.count) return;
    c.e = 0;
    do { if (++c.j >= p.group) return; c.count = row_of(c.j, c.first); } while (c.count == 0);
  };
  auto entry = [&](const Cursor& c) {
    return reinterpret_cast<const int2*>(p.tn_lut + (long long)(h0 + c.j) * p.tn_head_stride)[c.first + c.e];
  };
  Cursor pc;                                            // tid 0: the next entry to stage
  auto issue = [&](int f) {                             // one thread: stage flat entry f = (block id, query block)
    const int qb = entry(pc).y, qcol0 = (h0 + pc.j) * p.head_state;
    const uint32_t st = ring + (uint32_t)(f % ST) * STAGE_BYTES;
    uint64_t* bar = &full[f % ST];
    ptx::mbar_expect_tx(bar, STAGE_BYTES);
    for (int c = 0; c < CH; ++c) {
      ptx::tma_load_2d(st + c * BST_TILE, &maps.q, bar, qcol0 + c * 64, b * p.ctx_rows_q + qb * 64);
      ptx::tma_load_2d(st + T_BYTES + c * BST_TILE, &maps.dy, bar, qcol0 + c * 64, b * p.ctx_rows_q + qb * 64);
    }
    step(pc);
  };
  if (tid == 0) {
    ptx::mbar_init(&kvbar, 1);
    for (int e = 0; e < ST; ++e) ptx::mbar_init(&full[e], 1);
    ptx::fence_mbar_init();
  }
  __syncthreads();
  if (tid == 0 && total > 0) {
    ptx::mbar_expect_tx(&kvbar, 2 * T_BYTES);
    for (int c = 0; c < CH; ++c) {
      ptx::tma_load_2d(base + c * BST_TILE, &maps.k, &kvbar, col0 + c * 64, (int)krow0);
      ptx::tma_load_2d(vb + c * BST_TILE, &maps.v, &kvbar, col0 + c * 64, (int)krow0);
    }
    start(pc);
    for (int f = 0; f < total && f < ST; ++f) issue(f);
  }

  // This thread's two key rows r0, r0 + 8 of the block; its query columns are 8j + 2(lane%4) + x.
  const int r0 = warp * 16 + lane / 4;
  float dk[32], dv[32];
#pragma unroll
  for (int n = 0; n < 32; ++n) { dk[n] = 0.f; dv[n] = 0.f; }
  uint2 key = make_uint2(0u, 0u);
  unsigned long long call = 0;
  if constexpr (DROP) {
    const unsigned long long seed = (unsigned long long)p.seed_call[0];
    call = (unsigned long long)p.seed_call[1];
    key = make_uint2((unsigned)seed, (unsigned)(seed >> 32));
  }
  if (total > 0 && !ptx::mbar_wait(&kvbar, 0)) g_tc_error = 53;

  Cursor cc;                                            // every thread: the entry being computed
  start(cc);
  for (int e = 0; e < total; ++e, step(cc)) {
    const uint32_t st = ring + (uint32_t)(e % ST) * STAGE_BYTES;
    const int2 bq = entry(cc);
    const int h = h0 + cc.j;                            // its query head: mask, statistics and keep bits are h's
    const uint64_t* mask = p.mask ? p.mask + (p.mask_head_stride ? h * p.mask_head_stride : 0) : nullptr;
    if (tid < 64) {                                     // per query row t of the entry: its mask word and statistics
      const long long r = ((long long)b * p.heads + h) * p.ctx_rows_q + bq.y * 64 + tid;
      uint64_t w = ~0ull;
      if (mask) {
        w = mask[(long long)bq.x * 64 + tid];
        if (p.autoregress_at_key >= 0) w = autoregress_word<64>(w, p.autoregress_at_key, kb, bq.y * 64 + tid);
      }
      s_mask[tid] = w;
      s_m[tid] = p.row_max[r];
      s_il[tid] = 1.f / p.row_sum[r];
      s_d[tid] = p.delta[r];
      if constexpr (DROP) s_d[tid] *= p.keep_prob;
    }
    if (!ptx::mbar_wait(&full[e % ST], (uint32_t)(e / ST) & 1)) g_tc_error = 54;
    float s[32], dp[32];
#pragma unroll
    for (int n = 0; n < 32; ++n) { s[n] = 0.f; dp[n] = 0.f; }
    ptx::wg_fence();
#pragma unroll
    for (int c = 0; c < CH; ++c)
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
        ptx::wgmma_n64<BF16, 0, 0>(s, ptx::make_desc(base + c * BST_TILE + ks * 32, 16, 1024, ptx::SWZ_128B),
                                   ptx::make_desc(st + c * BST_TILE + ks * 32, 16, 1024, ptx::SWZ_128B));
        ptx::wgmma_n64<BF16, 0, 0>(dp, ptx::make_desc(vb + c * BST_TILE + ks * 32, 16, 1024, ptx::SWZ_128B),
                                   ptx::make_desc(st + T_BYTES + c * BST_TILE + ks * 32, 16, 1024, ptx::SWZ_128B));
      }
    ptx::wg_commit();
    if constexpr (DROP) {   // the entry's keep bits while the MMAs run: TPR neighbouring threads per query row
      constexpr int TPR = 2 * CH, GPT = 16 / TPR;       // GPT Philox blocks (4 keys each) per thread
      const int qr = tid / TPR, part = tid % TPR;
      const unsigned long long g0 =
          ((((unsigned long long)b * p.heads + h) * p.blocks + bq.x) * 64 + qr) * 16 + part * GPT;
      unsigned long long bits = 0;
#pragma unroll
      for (int u = 0; u < GPT; ++u)
        bits |= (unsigned long long)philox_keep4(g0 + u, call, key, p.keep_thr) << (4 * (part * GPT + u));
#pragma unroll
      for (int o = 1; o < TPR; o <<= 1) bits |= __shfl_xor_sync(0xffffffffu, bits, o);
      if (part == 0) s_keep[qr] = bits;
    }
    __syncthreads();                                    // the entry's mask words and statistics are in shared memory
    ptx::wg_wait<0>();
    ptx::wg_fence_regs(s);
    ptx::wg_fence_regs(dp);

    // s[4j + 2hh + x] = S^T[key r0 + 8hh][query q = 8j + 2(lane%4) + x]: scale, mask (bit key of word q), P^T, dS^T
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
      for (int x = 0; x < 2; ++x) {
        const int q = 8 * j + 2 * (lane % 4) + x;
        const uint64_t w = s_mask[q];
        const float mq = s_m[q], ilq = s_il[q], dq_ = s_d[q];
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          const int n = 4 * j + 2 * hh + x;
          float v = s[n] * p.scale;
          if (!((w >> (r0 + 8 * hh)) & 1ull)) v = -FLT_MAX;
          const float pr = exp2f((v - mq) * LOG2E) * ilq;
          if constexpr (DROP) {                         // dq_ = keep_prob D
            const bool keep = (s_keep[q] >> (r0 + 8 * hh)) & 1ull;
            s[n] = keep ? pr : 0.f;                     // (P o Z)^T
            dp[n] = (p.scale * p.rkeep) * (pr * ((keep ? dp[n] : 0.f) - dq_));   // dS^T
          } else {
            s[n] = pr;                                  // P^T
            dp[n] = p.scale * (pr * (dp[n] - dq_));     // dS^T
          }
        }
      }
    uint32_t a[4][4], g[4][4];
#pragma unroll
    for (int kk = 0; kk < 4; ++kk)
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        a[kk][r] = pack2<BF16>(s[8 * kk + 2 * r], s[8 * kk + 2 * r + 1]);
        g[kk][r] = pack2<BF16>(dp[8 * kk + 2 * r], dp[8 * kk + 2 * r + 1]);
      }
    ptx::wg_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {   // dO and Q = [64 queries = K][64 state columns of this warpgroup = N], MN-major
      ptx::wgmma_rs_n64<BF16, 1>(dv, a[kk], ptx::make_desc(st + T_BYTES + wg * BST_TILE + kk * 2048, BST_TILE, 1024, ptx::SWZ_128B));
      ptx::wgmma_rs_n64<BF16, 1>(dk, g[kk], ptx::make_desc(st + wg * BST_TILE + kk * 2048, BST_TILE, 1024, ptx::SWZ_128B));
    }
    ptx::wg_commit();
    ptx::wg_wait<0>();
    ptx::wg_fence_regs(dv);
    ptx::wg_fence_regs(dk);
    __syncthreads();                                    // every warp's MMAs that read this stage have retired
    if (tid == 0 && e + ST < total) issue(e + ST);
  }

  // epilogue: dK and dV summed over the group, rounded once (a key block no query of the group sees writes zeros)
  if constexpr (DROP) {
#pragma unroll
    for (int n = 0; n < 32; ++n) dv[n] *= p.rkeep;
  }
  const long long off = krow0 * SKV + col0 + wg * 64;
  store_rows<BF16>(reinterpret_cast<uint16_t*>(p.dk) + off, SKV, r0, lane, dk);
  store_rows<BF16>(reinterpret_cast<uint16_t*>(p.dv) + off, SKV, r0, lane, dv);
}

// ------------------------------------------------------------------------------------------------
// Envelope of the backward (the forward's, over every 16-bit tensor it touches); TC_NOT_APPLICABLE with the reason in
// bsmm_last_error() otherwise.
inline bool bst_attention_grad_applicable(int dtype, int bsize, int head_state, const void* const (&t)[8]) {
  uintptr_t any = 0;
  for (const void* x : t) any |= (uintptr_t)x;
  if (any & 15) { fail(0, "pointers must be 16-byte aligned for TMA"); return false; }
  return bst_tc_applicable(dtype, bsize, head_state, t[0], t[1], t[2]);
}

inline int tc_bst_attention_grad(int dtype, int bsize, const int32_t* nn_lut, const int32_t* tn_lut,
                                 const int32_t* tn_order, int lut_heads, int blocks, const void* mask, int mask_heads,
                                 int autoregress_at_key, const void* q, const void* k, const void* v, const void* o,
                                 const void* dy, const float* row_max, const float* row_sum, float* delta, void* dq,
                                 void* dk, void* dv, float scale, int batch, int heads, int head_state, int ctx_blks_q,
                                 int ctx_blks_k, cudaStream_t s, const BstAttnDrop* drop = nullptr, int kv_heads = 0) {
  const void* const all[8] = {q, k, v, o, dy, dq, dk, dv};
  if (!bst_attention_grad_applicable(dtype, bsize, head_state, all)) return TC_NOT_APPLICABLE;
  if (kv_heads <= 0) kv_heads = heads;                  // k, v, dk and dv are (batch, ctx_k, kv_heads * head_state)
  const uint64_t S = (uint64_t)heads * head_state, SKV = (uint64_t)kv_heads * head_state;
  BstAttnBwdTmaps maps;
  if (int e = cached_tmap_2d(&maps.q, dtype, q, S, (uint64_t)batch * ctx_blks_q * 64, S, 64, 64, CU_TENSOR_MAP_SWIZZLE_128B)) return e;
  if (int e = cached_tmap_2d(&maps.dy, dtype, dy, S, (uint64_t)batch * ctx_blks_q * 64, S, 64, 64, CU_TENSOR_MAP_SWIZZLE_128B)) return e;
  if (int e = cached_tmap_2d(&maps.k, dtype, k, SKV, (uint64_t)batch * ctx_blks_k * 64, SKV, 64, 64, CU_TENSOR_MAP_SWIZZLE_128B)) return e;
  if (int e = cached_tmap_2d(&maps.v, dtype, v, SKV, (uint64_t)batch * ctx_blks_k * 64, SKV, 64, 64, CU_TENSOR_MAP_SWIZZLE_128B)) return e;
  BstAttnBwdParams p;
  p.nn_lut = nn_lut; p.tn_lut = tn_lut; p.tn_order = tn_order;
  p.nn_head_stride = lut_heads > 1 ? 2LL * (ctx_blks_q + blocks) : 0;
  p.tn_head_stride = lut_heads > 1 ? 2LL * (ctx_blks_k + blocks) : 0;
  p.order_head_stride = lut_heads > 1 ? ctx_blks_k : 0;
  p.mask = reinterpret_cast<const uint64_t*>(mask);
  p.mask_head_stride = (mask && mask_heads > 1) ? (long long)blocks * 64 : 0;
  p.autoregress_at_key = autoregress_at_key; p.scale = scale;
  p.n_q = ctx_blks_q; p.n_k = ctx_blks_k; p.batch = batch; p.heads = heads; p.head_state = head_state;
  p.ctx_rows_q = ctx_blks_q * 64; p.ctx_rows_k = ctx_blks_k * 64;
  p.o = o; p.dy = dy; p.row_max = row_max; p.row_sum = row_sum; p.delta = delta;
  p.dq = dq; p.dk = dk; p.dv = dv;
  set_drop(p, drop);
  p.blocks = blocks;
  p.kv_heads = kv_heads; p.group = heads / kv_heads;
  const int ch = head_state / 64;
  const size_t smem = (size_t)(2 + 2 * BST_BWD_STAGES) * ch * BST_TILE + SMEM_ALIGN_SLACK;
  const unsigned grid_q = (unsigned)((long long)batch * heads * ctx_blks_q);
  const unsigned grid_k = (unsigned)((long long)batch * kv_heads * ctx_blks_k);
#define BSMM_LAUNCH_BWD(BFV, CHV, DRV)                                                   \
  { auto kq = wgmma_bst_attention_bwd_dq<BFV, CHV, DRV>;                                 \
    auto kk = wgmma_bst_attention_bwd_dkdv<BFV, CHV, DRV>;                               \
    static thread_local uint64_t cfg_q = 0, cfg_k = 0;                                   \
    if (int e = ensure_dyn_smem(kq, smem, cfg_q)) return e;                              \
    if (int e = ensure_dyn_smem(kk, smem, cfg_k)) return e;                              \
    kq<<<grid_q, BST_THREADS, smem, s>>>(p, maps);                                       \
    if (int e = check_launch(DRV ? "wgmma_bst_attention_bwd_dq_dropout" : "wgmma_bst_attention_bwd_dq")) return e; \
    kk<<<grid_k, BST_THREADS * CHV, smem, s>>>(p, maps); }
#define BSMM_LAUNCH_BWD_CH(BFV, DRV) \
  { if (ch == 2) BSMM_LAUNCH_BWD(BFV, 2, DRV) else BSMM_LAUNCH_BWD(BFV, 1, DRV) }
  const bool bf = dtype == BSMM_BF16;
  if (drop) { if (bf) BSMM_LAUNCH_BWD_CH(true, true) else BSMM_LAUNCH_BWD_CH(false, true) }
  else { if (bf) BSMM_LAUNCH_BWD_CH(true, false) else BSMM_LAUNCH_BWD_CH(false, false) }
#undef BSMM_LAUNCH_BWD_CH
#undef BSMM_LAUNCH_BWD
  return check_launch(drop ? "wgmma_bst_attention_bwd_dkdv_dropout" : "wgmma_bst_attention_bwd_dkdv");
}

}  // namespace bsmm
