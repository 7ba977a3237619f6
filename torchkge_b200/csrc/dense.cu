// Dense-score side paths: RESCAL's relation case and ranking / top-k over a small dense score matrix.
//
// RESCAL relation prediction (bilinear.py:115-121): the candidates are the relation MATRICES, so
// every (fact, relation) pair has its own vector  hr = h^T M_c  (batched matmul over b * n_rel
// (1 x d)(d x d) products) before the usual  (hr * t).sum(dim=2).  There is no shared candidate
// table to scan; the (n, n_rel) score matrix is small (n_rel relations) and is produced densely,
// in the reference's arithmetic: rescal_query_component (oneMKL order) then the ATen cascade sum.
#include "kernels.h"
#include "ptx.cuh"

namespace kge {

namespace {

constexpr int RR_THREADS = 256;
constexpr int RR_ITILE = 8;   // facts per CTA: one warp finishes one fact's score

// grid (n_rel, ceil(n / RR_ITILE)).  Thread t owns columns j = t, t + 256, ... of hr for the
// CTA's RR_ITILE facts: M_c[k][j] is loaded once per (k, j) and used for all of them.
__global__ void __launch_bounds__(RR_THREADS)
    rescal_rel_scores_kernel(const float* __restrict__ hrows, const float* __restrict__ trows,
                             const float* __restrict__ rel_mat, int dim, long long n, long long n_rel,
                             float* __restrict__ scores) {
  extern __shared__ float sm[];       // [RR_ITILE][dim] h rows, then [RR_ITILE][dim] hr
  float* sh = sm;
  float* shr = sm + (size_t)RR_ITILE * dim;
  const long long c = blockIdx.x;
  const long long i0 = (long long)blockIdx.y * RR_ITILE;
  const float* M = rel_mat + (size_t)c * dim * dim;
  for (int x = threadIdx.x; x < RR_ITILE * dim; x += RR_THREADS) {
    const long long i = i0 + x / dim;
    sh[x] = i < n ? hrows[(size_t)i * dim + x % dim] : 0.f;
  }
  __syncthreads();
  for (int j = threadIdx.x; j < dim; j += RR_THREADS) {
#pragma unroll
    for (int il = 0; il < RR_ITILE; ++il)
      shr[(size_t)il * dim + j] = rescal_query_component(true, dim, j, sh + (size_t)il * dim, M);
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long i = i0 + warp;     // RR_THREADS / 32 == RR_ITILE
  if (i >= n) return;
  const float* hr = shr + (size_t)warp * dim;
  const float* t = trows + (size_t)i * dim;
  float s;
  if (dim < 8) s = pair_score_natural<EL_DOT1>(dim, hr, hr, t, t);
  else s = pair_score_chains<EL_DOT1>(dim, hr, hr, t, t, lane);
  if (lane == 0) scores[(size_t)i * n_rel + c] = s;
}

// TransH relation case (interfaces.py:261-272 with the projections of translation.py:253-254): grid
// (n_rel, ceil(n / warps)), one warp per (fact i, relation c).  The warp projects h_i and t_i on the
// hyperplane of relation c into its shared-memory rows, then scores -||(P_c(h) + r_c) - P_c(t)||^2 in the
// L2-norm order: EL_L2_HEAD with candidate P_c(h), query planes (r_c, P_c(t)).
__global__ void transh_rel_scores_kernel(const float* __restrict__ hrows, const float* __restrict__ trows,
                                         const float* __restrict__ rel, const float* __restrict__ norm_vect,
                                         int dim, long long n, long long n_rel, float* __restrict__ scores) {
  extern __shared__ float sm[];       // per warp: [dim] P_c(h), then [dim] P_c(t)
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long c = blockIdx.x;
  const long long i = (long long)blockIdx.y * (blockDim.x >> 5) + warp;
  if (i >= n) return;
  float* ph = sm + (size_t)warp * 2 * dim;
  float* pt = ph + dim;
  const float* w = norm_vect + (size_t)c * dim;
  const float* r = rel + (size_t)c * dim;
  const float* h = hrows + (size_t)i * dim;
  const float* t = trows + (size_t)i * dim;
  float nh, nt;
  if (dim < 8) {
    nh = pair_score_natural<EL_DOT1>(dim, h, h, w, w);
    nt = pair_score_natural<EL_DOT1>(dim, t, t, w, w);
  } else {
    nh = pair_score_chains<EL_DOT1>(dim, h, h, w, w, lane);
    nt = pair_score_chains<EL_DOT1>(dim, t, t, w, w, lane);
  }
  for (int k = lane; k < dim; k += 32) {
    ph[k] = transh_project_elem(h[k], nh, w[k]);
    pt[k] = transh_project_elem(t[k], nt, w[k]);
  }
  __syncwarp();
  const float s = pair_score_chains<EL_L2_HEAD>(dim, r, pt, ph, ph, lane);
  if (lane == 0) scores[(size_t)i * n_rel + c] = s;
}

// TransD relation case (interfaces.py:261-272 with the projections of translation.py:645-646), laid out as
// transh_rel_scores_kernel: hrows / trows hold the first dim (= rel_emb_dim) coordinates of the raw entity
// rows and hs / ts their scalars s, so P_c(e)[j] = transd_project_elem(e[j], s_e, rel_proj[c][j]).
__global__ void transd_rel_scores_kernel(const float* __restrict__ hrows, const float* __restrict__ hs,
                                         const float* __restrict__ trows, const float* __restrict__ ts,
                                         const float* __restrict__ rel, const float* __restrict__ rel_proj,
                                         int dim, long long n, long long n_rel, float* __restrict__ scores) {
  extern __shared__ float sm[];       // per warp: [dim] P_c(h), then [dim] P_c(t)
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long c = blockIdx.x;
  const long long i = (long long)blockIdx.y * (blockDim.x >> 5) + warp;
  if (i >= n) return;
  float* ph = sm + (size_t)warp * 2 * dim;
  float* pt = ph + dim;
  const float* rp = rel_proj + (size_t)c * dim;
  const float* r = rel + (size_t)c * dim;
  const float* h = hrows + (size_t)i * dim;
  const float* t = trows + (size_t)i * dim;
  const float sh = hs[i], st = ts[i];
  for (int k = lane; k < dim; k += 32) {
    ph[k] = transd_project_elem(h[k], sh, rp[k]);
    pt[k] = transd_project_elem(t[k], st, rp[k]);
  }
  __syncwarp();
  const float s = pair_score_chains<EL_L2_HEAD>(dim, r, pt, ph, ph, lane);
  if (lane == 0) scores[(size_t)i * n_rel + c] = s;
}

// Grid of the per-relation projection kernels above: up to 8 warps (facts) per CTA within 48 KB of shared
// memory, one warp past dim 6144.  launch(grid, threads, smem, i_off) enqueues the facts from i_off on.
template <auto Kernel, typename Launch>
cudaError_t launch_projected_rel_scores(int dim, int64_t n, int64_t n_rel, Launch launch) {
  if (n <= 0 || n_rel <= 0) return cudaSuccess;
  const size_t per_warp = (size_t)2 * dim * sizeof(float);
  long long warps = (long long)(48 * 1024 / per_warp);
  warps = warps < 1 ? 1 : (warps > 8 ? 8 : warps);
  const size_t smem = (size_t)warps * per_warp;
  if (smem > 200 * 1024) return cudaErrorInvalidValue;
  if (smem > 48 * 1024) {
    const cudaError_t e = set_attribute_once<Kernel>(cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    if (e != cudaSuccess) return e;
  }
  const long long i_tiles = (n + warps - 1) / warps;
  for (long long y0 = 0; y0 < i_tiles; y0 += 65535) {     // gridDim.y limit
    const long long ny = i_tiles - y0 < 65535 ? i_tiles - y0 : 65535;
    launch(dim3((unsigned)n_rel, (unsigned)ny), (unsigned)(32 * warps), smem, y0 * warps);
  }
  return cudaGetLastError();
}

// One warp per row of a dense (n, n_c) score matrix:
//   raw_count[i] += #{c : s[i][c] >= s_true(i)},
//   filt_sub[i]  += sum over the row's CSR entries of [s[i][c] >= s_true(i)] - [s_true(i) == -inf]
// (get_rank, utils/operations.py:37-61, and filter_scores, utils/modeling.py:91-102, on a matrix that
// is small enough to exist).  s_true(i) = true_score_in[i] if given, else s[i][true_idx[i]].
__global__ void rank_dense_kernel(const float* __restrict__ scores, long long n, long long n_c,
                                  const int64_t* __restrict__ true_idx, const float* __restrict__ true_score_in,
                                  const int64_t* __restrict__ offs, const int64_t* __restrict__ ids,
                                  int32_t* __restrict__ raw_count, int32_t* __restrict__ filt_sub,
                                  float* __restrict__ true_score_out) {
  const long long i = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (i >= n) return;
  const float* row = scores + (size_t)i * n_c;
  const float st = true_score_in ? true_score_in[i] : row[true_idx[i]];
  int cnt = 0, sub = 0;
  for (long long c = lane; c < n_c; c += 32) cnt += row[c] >= st ? 1 : 0;
  if (offs) {
    for (long long e = offs[i] + lane; e < offs[i + 1]; e += 32) {
      const long long c = ids[e];
      if (c >= 0 && c < n_c) sub += (row[c] >= st ? 1 : 0) - (st == -INFINITY ? 1 : 0);
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
    sub += __shfl_xor_sync(0xffffffffu, sub, o);
  }
  if (lane == 0) {
    raw_count[i] += cnt;
    if (filt_sub) filt_sub[i] += sub;
    if (true_score_out) true_score_out[i] = st;
  }
}

__global__ void dense_to_pairs_kernel(const float* __restrict__ scores, long long total, long long n_c,
                                      int2* __restrict__ pairs) {
  const long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (gid >= total) return;
  pairs[gid] = make_int2(__float_as_int(scores[gid]), (int)(gid % n_c));
}

}  // namespace

cudaError_t launch_rescal_rel_scores(const float* hrows, const float* trows, const float* rel_mat, int dim,
                                     int64_t n, int64_t n_rel, float* scores, cudaStream_t stream) {
  if (n <= 0 || n_rel <= 0) return cudaSuccess;
  const size_t smem = (size_t)2 * RR_ITILE * dim * sizeof(float);
  if (smem > 200 * 1024) return cudaErrorInvalidValue;
  if (smem > 48 * 1024) {
    const cudaError_t e =
        set_attribute_once<rescal_rel_scores_kernel>(cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    if (e != cudaSuccess) return e;
  }
  const long long i_tiles = (n + RR_ITILE - 1) / RR_ITILE;
  for (long long y0 = 0; y0 < i_tiles; y0 += 65535) {     // gridDim.y limit
    const long long ny = i_tiles - y0 < 65535 ? i_tiles - y0 : 65535;
    dim3 grid((unsigned)n_rel, (unsigned)ny);
    const long long i_off = y0 * RR_ITILE;
    rescal_rel_scores_kernel<<<grid, RR_THREADS, smem, stream>>>(hrows + (size_t)i_off * dim, trows + (size_t)i_off * dim,
                                                               rel_mat, dim, n - i_off, n_rel,
                                                               scores + (size_t)i_off * n_rel);
  }
  return cudaGetLastError();
}

cudaError_t launch_transh_rel_scores(const float* hrows, const float* trows, const float* rel,
                                     const float* norm_vect, int dim, int64_t n, int64_t n_rel, float* scores,
                                     cudaStream_t stream) {
  return launch_projected_rel_scores<transh_rel_scores_kernel>(
      dim, n, n_rel, [&](dim3 grid, unsigned threads, size_t smem, long long i_off) {
        transh_rel_scores_kernel<<<grid, threads, smem, stream>>>(
            hrows + (size_t)i_off * dim, trows + (size_t)i_off * dim, rel, norm_vect, dim, n - i_off, n_rel,
            scores + (size_t)i_off * n_rel);
      });
}

cudaError_t launch_transd_rel_scores(const float* hrows, const float* hs, const float* trows, const float* ts,
                                     const float* rel, const float* rel_proj, int dim, int64_t n, int64_t n_rel,
                                     float* scores, cudaStream_t stream) {
  return launch_projected_rel_scores<transd_rel_scores_kernel>(
      dim, n, n_rel, [&](dim3 grid, unsigned threads, size_t smem, long long i_off) {
        transd_rel_scores_kernel<<<grid, threads, smem, stream>>>(
            hrows + (size_t)i_off * dim, hs + i_off, trows + (size_t)i_off * dim, ts + i_off, rel, rel_proj, dim,
            n - i_off, n_rel, scores + (size_t)i_off * n_rel);
      });
}

cudaError_t launch_rank_dense(const float* scores, int64_t n, int64_t n_c, const int64_t* true_idx,
                              const float* true_score_in, const int64_t* offs, const int64_t* ids,
                              int32_t* raw_count, int32_t* filt_sub, float* true_score_out, cudaStream_t stream) {
  if (n <= 0) return cudaSuccess;
  rank_dense_kernel<<<(unsigned)((n * 32 + 255) / 256), 256, 0, stream>>>(scores, n, n_c, true_idx, true_score_in, offs,
                                                                          ids, raw_count, filt_sub, true_score_out);
  return cudaGetLastError();
}

cudaError_t launch_dense_to_pairs(const float* scores, int64_t n, int64_t n_c, int2* pairs, cudaStream_t stream) {
  const long long total = (long long)n * n_c;
  if (total <= 0) return cudaSuccess;
  dense_to_pairs_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(scores, total, n_c, pairs);
  return cudaGetLastError();
}

}  // namespace kge
