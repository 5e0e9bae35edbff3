// Block-sparse attention decode: the attention of n new query rows (1 <= n <= bs) of each batch entry against a key /
// value cache, for sampling a trained Sparse Transformer one token (or one chunk) at a time.  Row r = positions[b] + i
// of batch entry b is row r of bst_attention over the cache: scaled scores, the mask word of the LUT entry's block id
// (with the autoregress_at_key rewrite), -FLT_MAX for masked keys, fp32 online softmax, P entering P V in the input
// dtype.  No reference launcher corresponds to it.
//
// Valid keys: only cache rows < L_b = min(positions[b] + n, ctx_rows_k) exist.  Rows at or beyond L_b are never read:
// their K and V tiles are zero-filled in shared memory by the copy itself (cp.async with a source size of 0), and
// their scores are -inf, so they get probability exactly 0 whatever the cache holds there (NaN and Inf included).  A
// row whose valid keys are all masked gets uniform weights over its valid keys; a row with no valid key, or an empty
// LUT row, is written as zeros.  positions[b] < 0 or positions[b] + n > ctx_rows_q writes NaN rows for entry b.
//
// Split rule: the LUT row of query block qb is cut into splits of DECODE_SPLIT consecutive entries, split s holding
// entries [s E, min((s + 1) E, count)).  It depends on the layout only, so a row's bits depend on nothing but the
// layout, the mask, its q and the valid cache -- not on batch, n, the other rows or their positions.
//   bst_attention_decode          one CTA per (split, touched query block t in {0, 1}, head, batch entry): the chunk's
//                                 rows of that block, padded to 16-row tiles (warp w owns block rows 16w..16w+15), walk
//                                 the split's entries through a DECODE_STAGES ring of cp.async copies; S = Q K^T and
//                                 O += P V on mma.sync.m16n8k16 (fp32 accumulators), K through ldmatrix, V through
//                                 ldmatrix.trans, P re-packed in registers as the A operand.  It stores the fp32
//                                 partial (m, l, O) of each of its rows to the workspace.
//   bst_attention_decode_combine  one warp per (batch entry, row, head): o = sum_s e^(m_s - M) O_s / sum_s e^(m_s - M) l_s
//                                 over the row's splits in split order, rounded once to the input dtype.
// Workspace: float2 (m, l) [batch][heads][nsplit][n], then float O [batch][heads][nsplit][n][head_state], with
// nsplit = ceil(nn_max / DECODE_SPLIT).  No atomics, no counters: every call overwrites what it reads.
//
// Grouped-query attention (caches of kv_heads < heads heads, g = heads / kv_heads, query head h reading kv head h / g):
// with a shared layout every head of a group walks the same LUT rows over the same K and V, so one CTA per (split, t,
// head slice, kv head, batch entry) stages each K / V tile once for a slice of hp = min(g, 64 / n) query heads.  Its
// DECODE_SLOTS = 64 row slots (4 warps x 16) hold the chunk's rows of each head in turn, slot j n + (r - r_lo) being
// block row r of head hfirst + j: rows of different heads are M rows of the same mma.sync, each with its own mask
// word, online softmax and partial.  A row's arithmetic does not depend on its slot, so its bits are those of the kernel above on
// the expanded cache.  Per-head layouts, and n too large to stack two heads, run hp = 1: one CTA per query head, in
// the row slots above, reading kv head h / g.  The combine is unchanged.
#pragma once
#include <float.h>
#include <algorithm>
#include "softmax.cuh"
#include "tc.cuh"

namespace bsmm {

constexpr int DECODE_SPLIT = 4;          // LUT entries per split
constexpr int DECODE_STAGES = 2;         // (K, V) tiles in flight per CTA
constexpr int DECODE_THREADS = 128;
constexpr int DECODE_SLOTS = DECODE_THREADS / 32 * 16;   // row slots of a CTA: 16 rows per warp

namespace dptx {
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, bool valid) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(valid ? 16 : 0) : "memory");
}
__device__ __forceinline__ void cp_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void ldsm_x4(uint32_t (&r)[4], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t (&r)[4], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
// D[16 x 8] += A[16 x 16] B[16 x 8], fp32 accumulators: d[2h + e] = D[l/4 + 8h][2(l%4) + e]
template <bool BF16>
__device__ __forceinline__ void mma16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  if constexpr (BF16)
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
  else
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
}  // namespace dptx

struct BstDecodeParams {
  const int32_t* lut;              // nn_lut: [lut_heads][ctx_blks_q + blocks][2]
  long long lut_head_stride;
  const void* mask;                // uint{bs} [mask_heads][blocks][bs] or null
  long long mask_head_stride;      // words
  int autoregress_at_key;          // < 0: off
  const uint16_t *q, *k, *v;       // q (batch, n, S); caches (batch, ctx_rows_k, kv_heads*head_state)
  void* o;                         // (batch, n, S)
  const int32_t* positions;
  float scale;
  int n, heads, head_state, nsplit;
  int ctx_rows_q, ctx_rows_k;
  float2* ml;                      // workspace: [batch][heads][nsplit][n] (m, l)
  float* acc;                      //            [batch][heads][nsplit][n][head_state] O
  int kv_heads, group;             // query head h reads kv head h / group
  int hp, hslices;                 // query heads per CTA (> 1: stacked row slots), CTAs per group: ceil(group / hp)
};

// Byte offset of 16-byte chunk c of row r in a tile of HSP 16-bit columns; the XOR keeps the eight rows an ldmatrix
// reads at one column in eight different bank groups.
template <int HSP> __device__ __forceinline__ uint32_t dec_off(int r, int c) {
  return (uint32_t)(r * HSP * 2 + ((c ^ (r & 7)) << 4));
}

template <bool BF16, int BS, int HSP>
__global__ void __launch_bounds__(DECODE_THREADS)
bst_attention_decode(const BstDecodeParams p) {
  using MW = typename MaskWord<BS>::type;
  constexpr int CH = HSP / 8;                          // 16-byte chunks per tile row
  constexpr int NT = BS / 8;                           // key n-tiles of S
  constexpr uint32_t TILE = BS * HSP * 2;
  constexpr float LOG2E = 1.4426950408889634f;
  extern __shared__ __align__(16) uint8_t smem_raw[];
  const uint32_t base = ptx::smem_u32(smem_raw);       // Q tile, then DECODE_STAGES x (K tile, V tile)
  const int tid = threadIdx.x, warp = tid / 32, lane = tid % 32;
  unsigned x = blockIdx.x;
  const int s = (int)(x % (unsigned)p.nsplit); x /= (unsigned)p.nsplit;
  const int t = (int)(x % 2u); x /= 2u;
  const int hsl = (int)(x % (unsigned)p.hslices); x /= (unsigned)p.hslices;
  const int kvh = (int)(x % (unsigned)p.kv_heads), b = (int)(x / (unsigned)p.kv_heads);
  const int hfirst = kvh * p.group + hsl * p.hp;       // this CTA's query heads: hfirst .. hfirst + nh - 1
  const int nh = min(p.hp, p.group - hsl * p.hp);
  const bool stacked = p.hp > 1;
  const uint32_t QTILE = (stacked ? DECODE_SLOTS : BS) * HSP * 2;
  const int n = p.n, hs = p.head_state;
  const int pos = p.positions[b];
  if (pos < 0 || pos > p.ctx_rows_q - n) return;       // the combine writes NaN rows
  const int qb = pos / BS + t;
  const int r_lo = max(pos, qb * BS) - qb * BS, r_hi = min(pos + n, (qb + 1) * BS) - qb * BS;   // block rows of the chunk
  if (r_lo >= r_hi) return;
  const int32_t* lut = p.lut + hfirst * p.lut_head_stride;   // stacked: a shared layout, one LUT for every head
  const int count = lut[2 * qb + 1];
  const int e0 = s * DECODE_SPLIT;
  if (e0 >= count) return;                             // the combine reads ceil(count / E) splits only
  const int ne = min(DECODE_SPLIT, count - e0);
  const int2* ent = reinterpret_cast<const int2*>(lut) + lut[2 * qb] + e0;
  const int L = min(pos + n, p.ctx_rows_k);
  const long long S = (long long)p.heads * hs, SKV = (long long)p.kv_heads * hs;
  const long long kcol0 = (long long)kvh * hs;
  // Row slot rs holds block row slot_row(rs, j) of head hfirst + j; valid: a row of the chunk (else it is computed
  // from zeros and never stored).
  auto slot_row = [&](int rs, int& j, bool& valid) {
    if (!stacked) { j = 0; valid = rs >= r_lo && rs < r_hi; return rs; }
    j = rs / n;
    const int r = rs % n + r_lo;
    valid = j < nh && r < r_hi;
    return r;
  };

  // Q rows of the chunk; other rows and the columns past head_state are zeros
  for (int idx = tid; idx < (int)(QTILE / (HSP * 2)) * CH; idx += DECODE_THREADS) {
    const int rs = idx / CH, c = idx % CH;
    int j;
    bool ok;
    const int r = slot_row(rs, j, ok);
    ok = ok && c * 8 < hs;
    const uint16_t* src = ok ? p.q + ((long long)b * n + (qb * BS + r - pos)) * S + (long long)(hfirst + j) * hs + c * 8 : p.q;
    dptx::cp_async16(base + dec_off<HSP>(rs, c), src, ok);
  }
  auto issue = [&](int j) {                            // all threads: K and V tiles of entry j of the split
    const int kb = ent[j].y;
    const uint32_t st = base + QTILE + (uint32_t)(j % DECODE_STAGES) * 2 * TILE;
    for (int idx = tid; idx < BS * CH; idx += DECODE_THREADS) {
      const int r = idx / CH, c = idx % CH;
      const int key = kb * BS + r;
      const bool ok = key < L && c * 8 < hs;           // rows past L_b never leave global memory
      const long long off = ok ? ((long long)b * p.ctx_rows_k + key) * SKV + kcol0 + c * 8 : 0;
      dptx::cp_async16(st + dec_off<HSP>(r, c), p.k + off, ok);
      dptx::cp_async16(st + TILE + dec_off<HSP>(r, c), p.v + off, ok);
    }
  };
#pragma unroll
  for (int j = 0; j < DECODE_STAGES; ++j) {            // one commit group per stage, empty ones included
    if (j < ne) issue(j);
    dptx::cp_commit();
  }

  const bool active = stacked ? warp * 16 < nh * n    // this warp's 16 rows hold a row of the chunk
                              : warp * 16 < r_hi && warp * 16 + 16 > r_lo;
  const int g = lane / 4;
  int rj[2], rrow[2];                                  // this thread's two rows: head hfirst + rj, block row rrow
  bool rvalid[2];
  const MW* rmask[2];
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    rrow[hh] = slot_row(warp * 16 + g + 8 * hh, rj[hh], rvalid[hh]);
    rmask[hh] = p.mask ? reinterpret_cast<const MW*>(p.mask) + (long long)(hfirst + rj[hh]) * p.mask_head_stride : nullptr;
    if (stacked && !rvalid[hh]) rmask[hh] = nullptr;  // its block row may lie past the block
  }
  float o[HSP / 8][4];
#pragma unroll
  for (int i = 0; i < HSP / 8; ++i)
#pragma unroll
    for (int e = 0; e < 4; ++e) o[i][e] = 0.f;
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};   // l: this thread's part of the row sum

  for (int j = 0; j < ne; ++j) {
    dptx::cp_wait<DECODE_STAGES - 1>();
    __syncthreads();
    if (active) {
      const uint32_t kt = base + QTILE + (uint32_t)(j % DECODE_STAGES) * 2 * TILE, vt = kt + TILE;
      float sc[NT][4];
#pragma unroll
      for (int i = 0; i < NT; ++i)
#pragma unroll
        for (int e = 0; e < 4; ++e) sc[i][e] = 0.f;
#pragma unroll 1
      for (int ks = 0; ks < HSP / 16; ++ks) {
        if (ks * 16 < hs) {
          uint32_t a[4];
          dptx::ldsm_x4(a, base + dec_off<HSP>(warp * 16 + lane % 16, 2 * ks + lane / 16));
#pragma unroll
          for (int np = 0; np < NT / 2; ++np) {
            uint32_t kf[4];
            dptx::ldsm_x4(kf, kt + dec_off<HSP>(np * 16 + (lane / 16) * 8 + lane % 8, 2 * ks + ((lane / 8) & 1)));
            dptx::mma16816<BF16>(sc[2 * np], a, kf[0], kf[1]);
            dptx::mma16816<BF16>(sc[2 * np + 1], a, kf[2], kf[3]);
          }
        }
      }
      // scale, mask (bst_softmax's order), then the valid-key rule; sc[i][2hh + x] is key 8i + 2(lane%4) + x of
      // row slot 16 warp + g + 8hh, block row rrow[hh]
      const int2 bk = ent[j];
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const int rr = rrow[hh];
        uint64_t w = ~0ull;
        if (rmask[hh]) {
          w = (uint64_t)rmask[hh][(long long)bk.x * BS + rr];
          if (p.autoregress_at_key >= 0) w = autoregress_word<BS>(w, p.autoregress_at_key, bk.y, qb * BS + rr);
        }
#pragma unroll
        for (int i = 0; i < NT; ++i)
#pragma unroll
          for (int xx = 0; xx < 2; ++xx) {
            const int kc = 8 * i + 2 * (lane % 4) + xx;
            float& v = sc[i][2 * hh + xx];
            v *= p.scale;
            if (!((w >> kc) & 1ull)) v = -FLT_MAX;
            if (bk.y * BS + kc >= L) v = -INFINITY;
          }
      }
      // online softmax: the 4 lanes of a quad share a row
      float alpha[2];
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        float mx = m[hh];
#pragma unroll
        for (int i = 0; i < NT; ++i) mx = fmaxf(mx, fmaxf(sc[i][2 * hh], sc[i][2 * hh + 1]));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
        float acc = 0.f;
        if (mx == -INFINITY) {                           // no valid key yet: nothing enters O or l
          alpha[hh] = 1.f;
#pragma unroll
          for (int i = 0; i < NT; ++i) sc[i][2 * hh] = sc[i][2 * hh + 1] = 0.f;
        } else {
          alpha[hh] = exp2f((m[hh] - mx) * LOG2E);       // subtract first: -FLT_MAX * LOG2E overflows
#pragma unroll
          for (int i = 0; i < NT; ++i)
#pragma unroll
            for (int xx = 0; xx < 2; ++xx) {
              float& v = sc[i][2 * hh + xx];
              v = exp2f((v - mx) * LOG2E);
              acc += v;
            }
        }
        m[hh] = mx;
        l[hh] = l[hh] * alpha[hh] + acc;
      }
#pragma unroll
      for (int i = 0; i < HSP / 8; ++i)
#pragma unroll
        for (int e = 0; e < 4; ++e) o[i][e] *= alpha[e >> 1];
      // O += P V: P in the input dtype as the A fragments of the BS / 16 key slices
      uint32_t pa[BS / 16][4];
#pragma unroll
      for (int kk = 0; kk < BS / 16; ++kk) {
        pa[kk][0] = pack2<BF16>(sc[2 * kk][0], sc[2 * kk][1]);
        pa[kk][1] = pack2<BF16>(sc[2 * kk][2], sc[2 * kk][3]);
        pa[kk][2] = pack2<BF16>(sc[2 * kk + 1][0], sc[2 * kk + 1][1]);
        pa[kk][3] = pack2<BF16>(sc[2 * kk + 1][2], sc[2 * kk + 1][3]);
      }
#pragma unroll
      for (int np = 0; np < HSP / 16; ++np) {
        if (np * 16 < hs) {
#pragma unroll
          for (int kk = 0; kk < BS / 16; ++kk) {
            uint32_t vf[4];
            dptx::ldsm_x4_t(vf, vt + dec_off<HSP>(kk * 16 + ((lane / 8) & 1) * 8 + lane % 8, 2 * np + lane / 16));
            dptx::mma16816<BF16>(o[2 * np], pa[kk], vf[0], vf[1]);
            dptx::mma16816<BF16>(o[2 * np + 1], pa[kk], vf[2], vf[3]);
          }
        }
      }
    }
    __syncthreads();                                    // every warp is done with stage j % DECODE_STAGES
    if (j + DECODE_STAGES < ne) issue(j + DECODE_STAGES);
    dptx::cp_commit();
  }
  dptx::cp_wait<0>();
  if (!active) return;

  // partials of this warp's rows of the chunk: (m, full l) and the unnormalised O
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    float sum = l[hh];
    sum += __shfl_xor_sync(0xffffffffu, sum, 1);
    sum += __shfl_xor_sync(0xffffffffu, sum, 2);
    if (!rvalid[hh]) continue;
    const long long slot = (((long long)b * p.heads + hfirst + rj[hh]) * p.nsplit + s) * n + (qb * BS + rrow[hh] - pos);
    if (lane % 4 == 0) p.ml[slot] = make_float2(m[hh], sum);
    float* out = p.acc + slot * hs;
#pragma unroll
    for (int i = 0; i < HSP / 8; ++i) {
      const int col = 8 * i + 2 * (lane % 4);
      if (col < hs) *reinterpret_cast<float2*>(out + col) = make_float2(o[i][2 * hh], o[i][2 * hh + 1]);
    }
  }
}

template <bool BF16>
__global__ void __launch_bounds__(DECODE_THREADS)
bst_attention_decode_combine(const BstDecodeParams p, int bs, long long rows) {
  constexpr float LOG2E = 1.4426950408889634f;
  const long long row = (long long)blockIdx.x * (DECODE_THREADS / 32) + threadIdx.x / 32;   // ((b n + i) heads + h)
  if (row >= rows) return;
  const int lane = threadIdx.x % 32, hs = p.head_state, n = p.n;
  const int h = (int)(row % p.heads);
  const long long bi = row / p.heads;
  const int i = (int)(bi % n), b = (int)(bi / n);
  uint16_t* out = reinterpret_cast<uint16_t*>(p.o) + bi * p.heads * hs + (long long)h * hs;
  const int pos = p.positions[b];
  float acc[8][2];
#pragma unroll
  for (int c = 0; c < 8; ++c) acc[c][0] = acc[c][1] = 0.f;
  float inv = 0.f;
  if (pos < 0 || pos > p.ctx_rows_q - n) {
    inv = __int_as_float(0x7fc00000);                  // NaN rows: a bad position faults nothing
  } else {
    const int qb = (pos + i) / bs;
    const int count = p.lut[h * p.lut_head_stride + 2 * qb + 1];
    const int ns = min((count + DECODE_SPLIT - 1) / DECODE_SPLIT, p.nsplit);
    const long long slot0 = ((long long)b * p.heads + h) * p.nsplit * n + i;
    float M = -INFINITY;
    for (int s = 0; s < ns; ++s) M = fmaxf(M, p.ml[slot0 + (long long)s * n].x);
    if (M != -INFINITY) {                              // else: no valid key, the row is zeros
      float lsum = 0.f;
      for (int s = 0; s < ns; ++s) {
        const long long slot = slot0 + (long long)s * n;
        const float2 ml = p.ml[slot];
        const float wgt = exp2f((ml.x - M) * LOG2E);
        lsum += wgt * ml.y;
        const float* src = p.acc + slot * hs;
#pragma unroll
        for (int c = 0; c < 8; ++c) {
          const int col = 64 * c + 2 * lane;
          if (col < hs) {
            const float2 v = *reinterpret_cast<const float2*>(src + col);
            acc[c][0] += wgt * v.x;
            acc[c][1] += wgt * v.y;
          }
        }
      }
      inv = 1.f / lsum;
    }
  }
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    const int col = 64 * c + 2 * lane;
    if (col < hs) *reinterpret_cast<uint32_t*>(out + col) = pack2<BF16>(acc[c][0] * inv, acc[c][1] * inv);
  }
}

// ------------------------------------------------------------------------------------------------
inline long long bst_decode_nsplit(int nn_max) { return nn_max > 0 ? (nn_max + DECODE_SPLIT - 1) / DECODE_SPLIT : 0; }

inline size_t bst_decode_workspace(int nn_max, int batch, int heads, int head_state, int n) {
  return (size_t)bst_decode_nsplit(nn_max) * batch * heads * n * (head_state + 2) * sizeof(float);
}

// Arguments are checked by the caller (api.cu).
inline int tc_bst_attention_decode(int dtype, int bsize, const int32_t* nn_lut, int lut_heads, int blocks, int nn_max,
                                   const void* mask, int mask_heads, int autoregress_at_key, const void* q,
                                   const void* k_cache, const void* v_cache, void* o, const int32_t* positions, int n,
                                   float scale, int batch, int heads, int head_state, int ctx_blks_q, int ctx_blks_k,
                                   void* workspace, cudaStream_t s, int kv_heads = 0) {
  BstDecodeParams p;
  p.lut = nn_lut; p.lut_head_stride = lut_heads > 1 ? 2LL * (ctx_blks_q + blocks) : 0;
  p.mask = mask; p.mask_head_stride = (mask && mask_heads > 1) ? (long long)blocks * bsize : 0;
  p.autoregress_at_key = autoregress_at_key;
  p.q = (const uint16_t*)q; p.k = (const uint16_t*)k_cache; p.v = (const uint16_t*)v_cache; p.o = o;
  p.positions = positions; p.scale = scale;
  p.n = n; p.heads = heads; p.head_state = head_state; p.nsplit = (int)bst_decode_nsplit(nn_max);
  p.ctx_rows_q = ctx_blks_q * bsize; p.ctx_rows_k = ctx_blks_k * bsize;
  p.ml = (float2*)workspace;
  p.acc = (float*)((char*)workspace + (size_t)p.nsplit * batch * heads * n * sizeof(float2));
  if (kv_heads <= 0) kv_heads = heads;
  p.kv_heads = kv_heads; p.group = heads / kv_heads;
  // a shared layout stacks up to 64 / n heads of a group in one CTA's row slots; per-head layouts run one head per CTA
  p.hp = lut_heads == 1 ? std::min(p.group, DECODE_SLOTS / n) : 1;
  if (p.hp < 2) p.hp = 1;
  p.hslices = (p.group + p.hp - 1) / p.hp;
  const int q_rows = p.hp > 1 ? DECODE_SLOTS : bsize;   // rows of the Q tile
  const bool bf = dtype == BSMM_BF16;
  if (p.nsplit > 0) {
    const int hsp = head_state <= 64 ? 64 : head_state <= 128 ? 128 : 256;
    const unsigned grid = (unsigned)((long long)batch * kv_heads * p.hslices * 2 * p.nsplit);
#define BSMM_LAUNCH_DEC(BFV, BSV, HSV)                                                   \
    { auto kern = bst_attention_decode<BFV, BSV, HSV>;                                   \
      const size_t smem = (size_t)(q_rows + 2 * DECODE_STAGES * BSV) * HSV * 2;          \
      const size_t smem_max = (size_t)(std::max(DECODE_SLOTS, BSV) + 2 * DECODE_STAGES * BSV) * HSV * 2; \
      static thread_local uint64_t cfg = 0;                                              \
      if (int e = ensure_dyn_smem(kern, smem_max, cfg)) return e;                        \
      kern<<<grid, DECODE_THREADS, smem, s>>>(p); }
#define BSMM_LAUNCH_DEC_HS(BFV, BSV)                                                     \
    { if (hsp == 64) BSMM_LAUNCH_DEC(BFV, BSV, 64)                                       \
      else if (hsp == 128) BSMM_LAUNCH_DEC(BFV, BSV, 128)                                \
      else BSMM_LAUNCH_DEC(BFV, BSV, 256) }
#define BSMM_LAUNCH_DEC_BS(BFV)                                                          \
    { if (bsize == 16) BSMM_LAUNCH_DEC_HS(BFV, 16)                                       \
      else if (bsize == 32) BSMM_LAUNCH_DEC_HS(BFV, 32)                                  \
      else BSMM_LAUNCH_DEC_HS(BFV, 64) }
    if (bf) BSMM_LAUNCH_DEC_BS(true) else BSMM_LAUNCH_DEC_BS(false)
#undef BSMM_LAUNCH_DEC_BS
#undef BSMM_LAUNCH_DEC_HS
#undef BSMM_LAUNCH_DEC
    if (int e = check_launch("bst_attention_decode")) return e;
  }
  const long long rows = (long long)batch * n * heads;
  const unsigned cgrid = (unsigned)((rows + DECODE_THREADS / 32 - 1) / (DECODE_THREADS / 32));
  if (bf) bst_attention_decode_combine<true><<<cgrid, DECODE_THREADS, 0, s>>>(p, bsize, rows);
  else bst_attention_decode_combine<false><<<cgrid, DECODE_THREADS, 0, s>>>(p, bsize, rows);
  return check_launch("bst_attention_decode_combine");
}

}  // namespace bsmm
