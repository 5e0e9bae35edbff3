// Embedding lookup and its gradient (bsmm_embedding_lookup, bsmm_embedding_grad in include/bsmm_b200.h).
//
// Lookup: y[i, :] = emb[idx[i], :], a bit copy of the row, or zeros when idx[i] is outside [0, C). Each row is copied
// by a group of threads, 16 bytes per access where the row starts allow.
//
// Gradient, deterministic and without atomics:
//   1. keys[i] = idx[i], or C when it is out of range; a stable radix sort of (key, position i) over the
//      ceil(log2(C + 1)) low bits groups equal rows, positions ascending, invalid entries last;
//   2. the sorted entries are cut into chunks of EMB_CHUNK. Per chunk and column, each run of equal keys is summed
//      in fp32 in position order. A run that starts and ends inside the chunk is rounded into dw directly; the chunk's
//      first and last runs, when they go on into a neighbouring chunk, are written as fp32 partials instead;
//   3. every aligned group of EMB_GROUP chunks that lies inside one run which began before it gets the sum of its
//      chunks' partials, in chunk order, so a very common row is not added up by one thread chunk by chunk;
//   4. the chunk where such a run starts adds the partials of the chunks it covers, in chunk order, taking a group's
//      sum in place of the group's chunks, and rounds the sum into dw once.
// The chunks and groups depend on idx only, so dw is bitwise reproducible; rows no index hits are zero (a memset before step 2).
#pragma once
#include <cub/device/device_radix_sort.cuh>
#include "dense_softmax.cuh"

namespace bsmm {

constexpr int EMB_THREADS = 256;
constexpr int EMB_CHUNK = 32;
constexpr int EMB_GROUP = 32;     // chunks per second-level partial

// bit copy of rows: V is the access unit (uint4, or the 2- or 4-byte element); KV units per row
template <typename V>
__global__ void __launch_bounds__(EMB_THREADS) embedding_lookup_kernel(const V* emb, const void* idx, int itype, V* y,
                                                                      long long n, int C, int KV, int tpr) {
  const int rpc = EMB_THREADS / tpr;
  for (long long r = (long long)blockIdx.x * rpc + threadIdx.x / tpr; r < n; r += (long long)gridDim.x * rpc) {
    const long long id = xent_label(idx, itype, r);
    const bool ok = id >= 0 && id < C;
    const V* src = emb + (ok ? id : 0) * KV;
    V* dst = y + r * KV;
    for (int c = threadIdx.x % tpr; c < KV; c += tpr) dst[c] = ok ? __ldg(src + c) : V{};
  }
}

inline int emb_tpr(int KV) {
  int t = 1;
  while (t < KV && t < EMB_THREADS) t *= 2;
  return t;
}

template <typename V>
int launch_embedding_lookup(const void* emb, const void* idx, int itype, void* y, long long n, int C, int KV,
                            cudaStream_t s) {
  const int tpr = emb_tpr(KV);
  const long long rpc = EMB_THREADS / tpr, blocks = (n + rpc - 1) / rpc;
  embedding_lookup_kernel<V><<<(unsigned)(blocks < (1 << 20) ? blocks : (1 << 20)), EMB_THREADS, 0, s>>>(
      reinterpret_cast<const V*>(emb), idx, itype, reinterpret_cast<V*>(y), n, C, KV, tpr);
  return check_launch("embedding_lookup");
}

struct EmbGradArgs {
  const void* dy;
  const uint32_t* keys;    // sorted
  const int32_t* pos;      // sorted with them
  void* dw;
  float* first;            // [chunks][K]: partial of the chunk's first run
  float* last;             // [chunks][K]: partial of its last run (when that is not also the first)
  float* group;            // [chunks / EMB_GROUP][K]: sums of `first` over groups inside one run
  long long n, chunks;
  int C, K;
};

__global__ void __launch_bounds__(EMB_THREADS) embedding_keys_kernel(const void* idx, int itype, long long n, int C,
                                                                     uint32_t* keys, int32_t* pos) {
  for (long long i = (long long)blockIdx.x * EMB_THREADS + threadIdx.x; i < n; i += (long long)gridDim.x * EMB_THREADS) {
    const long long id = xent_label(idx, itype, i);
    keys[i] = id >= 0 && id < C ? (uint32_t)id : (uint32_t)C;
    pos[i] = (int32_t)i;
  }
}

// thread (chunk, VEC columns); chunks of one CTA side by side
template <typename T, int VEC>
__global__ void __launch_bounds__(EMB_THREADS) embedding_grad_chunk_kernel(EmbGradArgs a, int tpr) {
  const int cv = blockIdx.y * tpr + threadIdx.x % tpr;
  const long long ch = (long long)blockIdx.x * (EMB_THREADS / tpr) + threadIdx.x / tpr;
  if (cv * VEC >= a.K || ch >= a.chunks) return;
  const int k0 = cv * VEC;
  const long long i0 = ch * EMB_CHUNK, i1 = min(i0 + EMB_CHUNK, a.n);
  const uint32_t before = i0 > 0 ? __ldg(a.keys + i0 - 1) : 0xffffffffu;
  const uint32_t after = i1 < a.n ? __ldg(a.keys + i1) : 0xffffffffu;
  uint32_t cur = __ldg(a.keys + i0);
  bool first = true;
  float s[VEC];
#pragma unroll
  for (int j = 0; j < VEC; ++j) s[j] = 0.f;
  auto flush = [&](bool ends) {
    const bool starts = !first || before != cur;
    if (starts && ends) {
      dsm_st<T, VEC>(reinterpret_cast<T*>(a.dw) + (long long)cur * a.K + k0, s);
    } else {
      float* p = (first ? a.first : a.last) + ch * a.K + k0;
#pragma unroll
      for (int j = 0; j < VEC; ++j) p[j] = s[j];
    }
  };
  for (long long i = i0; i < i1; ++i) {
    const uint32_t key = __ldg(a.keys + i);
    if (key >= (uint32_t)a.C) break;                 // invalid entries sort last
    if (key != cur) {
      flush(true);
      cur = key;
      first = false;
#pragma unroll
      for (int j = 0; j < VEC; ++j) s[j] = 0.f;
    }
    float v[VEC];
    dsm_ld<T, VEC, false>(reinterpret_cast<const T*>(a.dy) + (long long)__ldg(a.pos + i) * a.K + k0, v);
#pragma unroll
    for (int j = 0; j < VEC; ++j) s[j] += v[j];
  }
  // the run of `cur` goes on only if it fills the chunk's end and the next chunk starts with it
  if (cur < (uint32_t)a.C) flush(__ldg(a.keys + i1 - 1) != cur || after != cur);
}

// Group g holds entries [g * EMB_GROUP * EMB_CHUNK, (g + 1) * EMB_GROUP * EMB_CHUNK). It lies inside a run that began
// before it when the entry before it and its last entry share a valid key; then each of its chunks is that key only and
// wrote its whole sum to `first`.
__device__ __forceinline__ bool emb_group_in_run(const EmbGradArgs& a, long long g, uint32_t& key) {
  const long long e0 = g * EMB_GROUP * EMB_CHUNK, e1 = e0 + EMB_GROUP * EMB_CHUNK;
  if (e0 == 0 || e1 > a.n) return false;
  key = __ldg(a.keys + e1 - 1);
  return key < (uint32_t)a.C && __ldg(a.keys + e0 - 1) == key;
}

// thread (group, column): the group's sum of `first`, in chunk order
__global__ void __launch_bounds__(EMB_THREADS) embedding_grad_groups_kernel(EmbGradArgs a) {
  const long long g = blockIdx.x;
  const int k = blockIdx.y * EMB_THREADS + threadIdx.x;
  uint32_t key;
  if (k >= a.K || !emb_group_in_run(a, g, key)) return;
  float t = 0.f;
  for (long long c = g * EMB_GROUP; c < (g + 1) * EMB_GROUP; ++c) t += a.first[c * a.K + k];
  a.group[g * a.K + k] = t;
}

// thread (chunk, column): a chunk whose last run starts in it and goes on into the next chunk adds that run's partials
// in chunk order, a whole group at a time where the run covers one, and rounds the sum into dw
template <typename T>
__global__ void __launch_bounds__(EMB_THREADS) embedding_grad_runs_kernel(EmbGradArgs a) {
  const long long ch = blockIdx.x;
  const int k = blockIdx.y * EMB_THREADS + threadIdx.x;
  if (k >= a.K) return;
  const long long i0 = ch * EMB_CHUNK, i1 = min(i0 + EMB_CHUNK, a.n);
  const uint32_t key = __ldg(a.keys + i1 - 1);
  if (key >= (uint32_t)a.C || i1 == a.n || __ldg(a.keys + i1) != key) return;    // invalid, or the run ends here
  const bool single = __ldg(a.keys + i0) == key;
  if (single && i0 > 0 && __ldg(a.keys + i0 - 1) == key) return;                // the run started in an earlier chunk
  float t = (single ? a.first : a.last)[ch * a.K + k];
  for (long long c = ch + 1; c < a.chunks;) {
    uint32_t gkey;
    long long next;
    if (c % EMB_GROUP == 0 && emb_group_in_run(a, c / EMB_GROUP, gkey) && gkey == key) {
      t += a.group[(c / EMB_GROUP) * a.K + k];
      next = c + EMB_GROUP;
    } else {
      t += a.first[c * a.K + k];
      const long long e = min((c + 1) * EMB_CHUNK, a.n);
      if (__ldg(a.keys + e - 1) != key) break;
      next = c + 1;
    }
    const long long e = next * EMB_CHUNK;                       // first entry after what was added
    if (e >= a.n || __ldg(a.keys + e) != key) break;
    c = next;
  }
  reinterpret_cast<T*>(a.dw)[(long long)key * a.K + k] = from_f32<T>(t);
}

inline int emb_sort_bits(int C) {
  int b = 1;
  while (b < 32 && (1ull << b) <= (unsigned long long)C) ++b;   // keys 0..C fit in b bits
  return b;
}

inline size_t emb_align(size_t b) { return (b + 255) & ~(size_t)255; }

// workspace: keys and positions twice (sort input and output), the three partial arrays, then CUB's temporary storage
inline size_t emb_sort_temp_bytes(long long n, int C) {
  size_t t = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, t, (const uint32_t*)nullptr, (uint32_t*)nullptr, (const int32_t*)nullptr,
                                  (int32_t*)nullptr, (int)n, 0, emb_sort_bits(C));
  return t;
}

inline size_t emb_workspace_bytes(long long n, int C, int K) {
  const long long chunks = (n + EMB_CHUNK - 1) / EMB_CHUNK;
  return 4 * emb_align(n * 4) + 2 * emb_align((size_t)chunks * K * 4) + emb_align((size_t)(chunks / EMB_GROUP) * K * 4) +
         emb_align(emb_sort_temp_bytes(n, C));
}

template <typename T>
int launch_embedding_grad(const void* dy, const void* idx, int itype, void* dw, void* ws, long long n, int C, int K,
                          bool vec, cudaStream_t s) {
  char* p = reinterpret_cast<char*>(ws);
  uint32_t* keys_in = reinterpret_cast<uint32_t*>(p);  p += emb_align(n * 4);
  uint32_t* keys = reinterpret_cast<uint32_t*>(p);     p += emb_align(n * 4);
  int32_t* pos_in = reinterpret_cast<int32_t*>(p);     p += emb_align(n * 4);
  int32_t* pos = reinterpret_cast<int32_t*>(p);        p += emb_align(n * 4);
  EmbGradArgs a = {};
  a.chunks = (n + EMB_CHUNK - 1) / EMB_CHUNK;
  a.first = reinterpret_cast<float*>(p);               p += emb_align((size_t)a.chunks * K * 4);
  a.last = reinterpret_cast<float*>(p);                p += emb_align((size_t)a.chunks * K * 4);
  const long long groups = a.chunks / EMB_GROUP;
  a.group = reinterpret_cast<float*>(p);               p += emb_align((size_t)groups * K * 4);
  size_t temp = emb_sort_temp_bytes(n, C);
  const long long kb = (n + EMB_THREADS - 1) / EMB_THREADS;
  embedding_keys_kernel<<<(unsigned)(kb < 65536 ? kb : 65536), EMB_THREADS, 0, s>>>(idx, itype, n, C, keys_in, pos_in);
  if (int e = check_launch("embedding_grad")) return e;
  cudaError_t e = cub::DeviceRadixSort::SortPairs(p, temp, keys_in, keys, pos_in, pos, (int)n, 0, emb_sort_bits(C), s);
  if (e != cudaSuccess) { cudaGetLastError(); return fail((int)e, "embedding_grad: radix sort: %s", cudaGetErrorString(e)); }
  e = cudaMemsetAsync(dw, 0, (size_t)C * K * sizeof(T), s);
  if (e != cudaSuccess) { cudaGetLastError(); return fail((int)e, "embedding_grad: memset: %s", cudaGetErrorString(e)); }
  a.dy = dy; a.keys = keys; a.pos = pos; a.dw = dw; a.n = n; a.C = C; a.K = K;
  constexpr int V = 16 / sizeof(T);
  const int VEC = vec ? V : 1, tpr = emb_tpr(K / VEC);
  const dim3 grid((unsigned)((a.chunks + EMB_THREADS / tpr - 1) / (EMB_THREADS / tpr)), (unsigned)((K / VEC + tpr - 1) / tpr));
  if (vec) embedding_grad_chunk_kernel<T, V><<<grid, EMB_THREADS, 0, s>>>(a, tpr);
  else     embedding_grad_chunk_kernel<T, 1><<<grid, EMB_THREADS, 0, s>>>(a, tpr);
  if (int e2 = check_launch("embedding_grad")) return e2;
  if (groups > 0) {
    embedding_grad_groups_kernel<<<dim3((unsigned)groups, (unsigned)((K + EMB_THREADS - 1) / EMB_THREADS)), EMB_THREADS, 0, s>>>(a);
    if (int e3 = check_launch("embedding_grad")) return e3;
  }
  embedding_grad_runs_kernel<T><<<dim3((unsigned)a.chunks, (unsigned)((K + EMB_THREADS - 1) / EMB_THREADS)), EMB_THREADS, 0, s>>>(a);
  return check_launch("embedding_grad");
}

}  // namespace bsmm
