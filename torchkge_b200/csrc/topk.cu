// Top-k selection for EntityInference / RelationInference (torchkge/inference.py:78-250).
//
// The reference materialises the (b, n_candidates) score matrix, masks the known facts with -inf
// (filter_scores with true_idx = None, utils/modeling.py:91-102) and sorts every row.  Here the dense
// scan runs in "collect" mode (scan.cu): per query only the candidates whose exact score is not
// below the query's current k-th best are written out, chunk of candidate rows by chunk; after each
// chunk this kernel merges what was collected into the query's running top-k and raises the
// threshold.  Nothing of size (b, n_candidates) exists; after the first chunk a query collects
// ~k * chunk / rows_seen candidates per chunk.
//
// Order: scores descending, NaN above everything (as torch.topk / sort(descending=True) treat it),
// exact ties by ascending candidate id (the reference leaves the order among ties unspecified).
// The order is that of the score's bits (score_key): +0.0 ranks above -0.0 although they compare
// equal, so that the returned score keeps its sign bit.
//
// Ids are global: a scan over a shard of rows [ent_lo, ent_lo + n_rows) collects ent_lo + row, and
// the mask CSR lists global ids.  The per-shard lists are combined by topk_lists_merge_kernel under
// the same key order, which gives the unsharded result bit for bit (keys are unique, so the global
// top k lies in the union of the shards' top min(k, rows)).
#include "kernels.h"

namespace kge {

namespace {

constexpr int SORT_N = 2048;        // keys sorted per pass: the held k plus SORT_N - k new ones
constexpr int MERGE_THREADS = 256;

// monotone map float -> uint32 (larger float -> larger key), NaN on top
__device__ __forceinline__ unsigned score_key(float s) {
  unsigned u = __float_as_uint(s);
  if (s != s) return 0xffffffffu;
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float key_score(unsigned k) {
  if (k == 0xffffffffu) return __uint_as_float(0x7fc00000u);
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}
// 64-bit key: score key, then (0xffffffff - id) so that among equal scores the smaller id sorts first
// in descending order.  0 is reserved for "empty" (the smallest real key is -inf's, 0x007fffff << 32).
__device__ __forceinline__ unsigned long long make_key(float s, int id) {
  return ((unsigned long long)score_key(s) << 32) | (unsigned long long)(0xffffffffu - (unsigned)id);
}

// is `id` in the sorted range ids[lo, hi) ?
__device__ __forceinline__ bool masked(const int64_t* __restrict__ ids, long long lo, long long hi, long long id) {
  while (lo < hi) {
    const long long mid = (lo + hi) >> 1;
    const long long v = ids[mid];
    if (v == id) return true;
    if (v < id) lo = mid + 1; else hi = mid;
  }
  return false;
}

// descending bitonic sort of SORT_N keys in shared memory
__device__ void bitonic_desc(unsigned long long* keys) {
  for (int size = 2; size <= SORT_N; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      __syncthreads();
      for (int t = threadIdx.x; t < SORT_N / 2; t += MERGE_THREADS) {
        const int lo = 2 * t - (t & (stride - 1));
        const int hi = lo + stride;
        const bool desc = ((lo & size) == 0);
        const unsigned long long a = keys[lo], b = keys[hi];
        if ((a < b) == desc) { keys[lo] = b; keys[hi] = a; }
      }
    }
  }
  __syncthreads();
}

__global__ void __launch_bounds__(MERGE_THREADS)
    topk_merge_kernel(unsigned long long* __restrict__ best, int k, const int2* __restrict__ col_buf,
                      const unsigned* __restrict__ col_count, unsigned long long col_cap, long long dense_count,
                      const int64_t* __restrict__ mask_offs, const int64_t* __restrict__ mask_ids,
                      float* __restrict__ thr) {
  __shared__ unsigned long long keys[SORT_N];
  const long long q = blockIdx.x;
  unsigned long long cnt = dense_count >= 0 ? (unsigned long long)dense_count : (unsigned long long)col_count[q];
  if (cnt > col_cap) cnt = col_cap;
  unsigned long long* mine = best + (size_t)q * k;
  const int2* list = col_buf + (size_t)q * col_cap;
  const long long m_lo = mask_offs ? mask_offs[q] : 0, m_hi = mask_offs ? mask_offs[q + 1] : 0;
  const int fresh = SORT_N - k;     // new entries taken per pass
  if (cnt == 0) return;             // nothing collected: list and threshold stay as they are
  if (k <= 32 && cnt <= 128) {
    // the usual case after the first chunk: a handful of new candidates against a short list --
    // one warp keeps the list in registers (one key per lane, descending) and inserts one at a time
    if (threadIdx.x >= 32) return;
    const int lane = threadIdx.x;
    unsigned long long mykey = lane < k ? mine[lane] : 0ull;
    for (unsigned long long e = 0; e < cnt; ++e) {
      const int2 v = list[e];
      float s = __int_as_float(v.x);
      if (m_hi > m_lo && masked(mask_ids, m_lo, m_hi, (long long)v.y)) s = -INFINITY;
      const unsigned long long key = make_key(s, v.y);
      const unsigned ahead = __ballot_sync(0xffffffffu, lane < k && mykey > key);
      const int pos = __popc(ahead);                    // keys ahead of the new one keep their place
      if (pos >= k) continue;
      const unsigned long long up = __shfl_up_sync(0xffffffffu, mykey, 1);
      if (lane > pos) mykey = up;                       // everything behind moves down one slot
      if (lane == pos) mykey = key;
    }
    if (lane < k) mine[lane] = mykey;
    const unsigned long long kth = __shfl_sync(0xffffffffu, mykey, k - 1);
    if (lane == 0) thr[q] = kth == 0ull ? -INFINITY : key_score((unsigned)(kth >> 32));
    return;
  }
  for (unsigned long long t0 = 0; t0 < cnt; t0 += fresh) {
    for (int i = threadIdx.x; i < SORT_N; i += MERGE_THREADS) {
      unsigned long long key = 0ull;
      if (i < k) {
        key = mine[i];
      } else {
        const unsigned long long e = t0 + (unsigned long long)(i - k);
        if (e < cnt) {
          const int2 v = list[e];
          float s = __int_as_float(v.x);
          if (m_hi > m_lo && masked(mask_ids, m_lo, m_hi, (long long)v.y)) s = -INFINITY;
          key = make_key(s, v.y);
        }
      }
      keys[i] = key;
    }
    bitonic_desc(keys);
    for (int i = threadIdx.x; i < k; i += MERGE_THREADS) mine[i] = keys[i];
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    const unsigned long long kth = keys[k - 1];
    thr[q] = kth == 0ull ? -INFINITY : key_score((unsigned)(kth >> 32));
  }
}

__global__ void topk_finish_kernel(const unsigned long long* __restrict__ best, int k, long long n_q,
                                   int64_t* __restrict__ pred, float* __restrict__ scores) {
  const long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (gid >= n_q * k) return;
  const unsigned long long key = best[gid];
  pred[gid] = key == 0ull ? -1 : (int64_t)(0xffffffffu - (unsigned)(key & 0xffffffffull));
  scores[gid] = key == 0ull ? -INFINITY : key_score((unsigned)(key >> 32));
}

// ---- merge of per-shard top-k lists (kge_topk_merge) ----
constexpr int LISTS_WARPS = 4;      // queries per block, one warp each

// key of entry `at` of a (pred, scores) list: the key the scan gave it, 0 for an empty slot (pred < 0)
__device__ __forceinline__ unsigned long long list_key(const int64_t* __restrict__ pred,
                                                       const float* __restrict__ scores, size_t at) {
  const int64_t id = pred[at];
  return id < 0 ? 0ull : make_key(scores[at], (int)id);
}

// One warp per query: lane l holds the heads of lists l and l + 32.  Every step takes the largest head
// (warp max of the 64-bit keys; keys are unique because ids are) and advances the list it came from.
// Lists are sorted best first, so the output is the k best keys of their union, in key order.
__global__ void __launch_bounds__(LISTS_WARPS * 32)
    topk_lists_merge_kernel(const int64_t* __restrict__ pred_in, const float* __restrict__ scores_in,
                            int n_lists, long long n, int k_in, int k, int64_t* __restrict__ pred,
                            float* __restrict__ scores) {
  const long long q = (long long)blockIdx.x * LISTS_WARPS + threadIdx.x / 32;
  if (q >= n) return;                // whole warps leave together
  const int lane = threadIdx.x & 31;
  const size_t list_stride = (size_t)n * k_in, row = (size_t)q * k_in;
  const size_t base0 = (size_t)lane * list_stride + row, base1 = (size_t)(lane + 32) * list_stride + row;
  int pos0 = 0, pos1 = 0;
  unsigned long long h0 = lane < n_lists ? list_key(pred_in, scores_in, base0) : 0ull;
  unsigned long long h1 = lane + 32 < n_lists ? list_key(pred_in, scores_in, base1) : 0ull;
  int64_t* out_pred = pred + (size_t)q * k;
  float* out_scores = scores + (size_t)q * k;
  for (int j = 0; j < k; ++j) {
    unsigned long long top = h0 > h1 ? h0 : h1;
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      const unsigned long long o = __shfl_xor_sync(0xffffffffu, top, off);
      top = o > top ? o : top;
    }
    if (top == 0ull) {               // every list is exhausted: the remaining slots stay empty
      for (int i = j + lane; i < k; i += 32) {
        out_pred[i] = -1;
        out_scores[i] = -INFINITY;
      }
      return;
    }
    if (lane == 0) {
      out_pred[j] = (int64_t)(0xffffffffu - (unsigned)(top & 0xffffffffull));
      out_scores[j] = key_score((unsigned)(top >> 32));
    }
    if (h0 == top) {
      ++pos0;
      h0 = pos0 < k_in ? list_key(pred_in, scores_in, base0 + pos0) : 0ull;
    } else if (h1 == top) {
      ++pos1;
      h1 = pos1 < k_in ? list_key(pred_in, scores_in, base1 + pos1) : 0ull;
    }
  }
}

}  // namespace

cudaError_t launch_topk_lists_merge(const int64_t* pred_in, const float* scores_in, int n_lists, int64_t n,
                                    int k_in, int k, int64_t* pred, float* scores, cudaStream_t stream) {
  if (n <= 0) return cudaSuccess;
  if (n_lists < 1 || n_lists > TOPK_MAX_LISTS || k < 1 || k > TOPK_MAX_K || k_in < 1) return cudaErrorInvalidValue;
  const long long blocks = (n + LISTS_WARPS - 1) / LISTS_WARPS;
  topk_lists_merge_kernel<<<(unsigned)blocks, LISTS_WARPS * 32, 0, stream>>>(pred_in, scores_in, n_lists, n, k_in,
                                                                             k, pred, scores);
  return cudaGetLastError();
}

cudaError_t launch_topk_merge(unsigned long long* best, int k, const int2* col_buf,
                              const unsigned* col_count, unsigned long long col_cap, long long dense_count,
                              const int64_t* mask_offs, const int64_t* mask_ids, float* thr, int64_t n_q,
                              cudaStream_t stream) {
  if (n_q <= 0) return cudaSuccess;
  if (k < 1 || k > TOPK_MAX_K) return cudaErrorInvalidValue;
  topk_merge_kernel<<<(unsigned)n_q, MERGE_THREADS, 0, stream>>>(best, k, col_buf, col_count, col_cap, dense_count,
                                                                mask_offs, mask_ids, thr);
  return cudaGetLastError();
}

cudaError_t launch_topk_finish(const unsigned long long* best, int k, int64_t n_q, int64_t* pred,
                               float* scores, cudaStream_t stream) {
  if (n_q <= 0) return cudaSuccess;
  const long long total = (long long)n_q * k;
  topk_finish_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(best, k, n_q, pred, scores);
  return cudaGetLastError();
}

}  // namespace kge
