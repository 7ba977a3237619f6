// Relation co-occurrence counts for the data-redundancy analysis (torchkge/utils/data_redundancy.py,
// Akrami et al., SIGMOD 2020): how many (h, t) entity pairs two relations share, in the same or in the
// reversed orientation.
//
// Both sides are sorted, deduplicated keys (h * n_ent + t) * n_rel + r cut into segments of equal
// (h, t); a segment holds distinct relations, so it has at most n_rel keys.  One warp takes one left
// segment: it bisects the right side's segment pairs for (h, t) -- or (t, h) when flipped -- and adds 1
// to counts[r_a][r_b] for every key r_a of the left segment and r_b of the right one, the lanes striding
// over the |left| x |right| products so that a pair carrying hundreds of relations is shared by the warp.
#include "kernels.h"

namespace kge {

namespace {

constexpr int CO_THREADS = 256;
constexpr int CO_WARPS = CO_THREADS / 32;
constexpr long long CO_MAX_CTAS = 1LL << 20;   // grid-stride beyond this

__global__ void __launch_bounds__(CO_THREADS)
    cooccurrence_kernel(const int64_t* __restrict__ lkeys, const int64_t* __restrict__ loffs,
                        const int64_t* __restrict__ lpairs, long long n_left, const int64_t* __restrict__ rkeys,
                        const int64_t* __restrict__ roffs, const int64_t* __restrict__ rpairs, long long n_right,
                        long long n_ent, long long n_rel, bool flip, bool upper,
                        unsigned long long* __restrict__ counts) {
  const int lane = threadIdx.x & 31;
  const long long stride = (long long)gridDim.x * CO_WARPS;
  for (long long s = (long long)blockIdx.x * CO_WARPS + (threadIdx.x >> 5); s < n_left; s += stride) {
    const long long p = lpairs[s];
    long long want = p;
    if (flip) {
      const long long h = p / n_ent;
      want = (p - h * n_ent) * n_ent + h;
    }
    long long lo = 0, hi = n_right;   // first right segment with pair >= want
    while (lo < hi) {
      const long long mid = (lo + hi) >> 1;
      if (rpairs[mid] < want) lo = mid + 1;
      else hi = mid;
    }
    if (lo == n_right || rpairs[lo] != want) continue;   // uniform over the warp
    const long long l0 = loffs[s], nl = loffs[s + 1] - l0;
    const long long r0 = roffs[lo], nr = roffs[lo + 1] - r0;
    const long long lbase = p * n_rel, rbase = want * n_rel;
    for (long long x = lane; x < nl * nr; x += 32) {
      const long long i = x / nr, j = x - i * nr;
      const long long ra = lkeys[l0 + i] - lbase, rb = rkeys[r0 + j] - rbase;
      if (!upper || ra < rb) atomicAdd(counts + ra * n_rel + rb, 1ULL);
    }
  }
}

}  // namespace

cudaError_t launch_cooccurrence(const int64_t* lkeys, const int64_t* loffs, const int64_t* lpairs, int64_t n_left,
                                const int64_t* rkeys, const int64_t* roffs, const int64_t* rpairs, int64_t n_right,
                                int64_t n_ent, int64_t n_rel, bool flip, bool upper, unsigned long long* counts,
                                cudaStream_t stream) {
  if (n_left <= 0 || n_right <= 0) return cudaSuccess;
  long long ctas = (n_left + CO_WARPS - 1) / CO_WARPS;
  if (ctas > CO_MAX_CTAS) ctas = CO_MAX_CTAS;
  cooccurrence_kernel<<<(unsigned)ctas, CO_THREADS, 0, stream>>>(lkeys, loffs, lpairs, n_left, rkeys, roffs, rpairs,
                                                                 n_right, n_ent, n_rel, flip, upper, counts);
  return cudaGetLastError();
}

}  // namespace kge
