// Internal launch interface between api.cu and the kernel translation units.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <type_traits>

#include "../../include/kge_b200.h"
#include "reduce.cuh"

namespace kge {

constexpr int TILE_Q = KGE_TILE_Q;  // queries per CTA tile
constexpr int TILE_C = KGE_TILE_C;  // candidates per CTA tile

// Three-plane models (KGE_ANALOGY) hand over planes 0 and 1 of a table; the planes are equally
// spaced in memory (include/kge_b200.h), so plane 2 follows from the two pointers.
__host__ __device__ inline const float* third_plane(const float* p0, const float* p1) {
  return p1 == nullptr ? nullptr : p1 + (p1 - p0);
}
__host__ __device__ inline float* third_plane(float* p0, float* p1) {
  return p1 == nullptr ? nullptr : p1 + (p1 - p0);
}

// model/side -> element kind (-1 if unsupported)
int elem_kind_for(int model, int side);
int elem_qw(int el);
int elem_cw(int el);

constexpr int SCAN_KC = 32;          // schedule positions per pipeline stage of the scan
constexpr int SCAN_MAX_DIM = 8192;   // schedule bytes carried in the kernel parameters

// Passed BY VALUE as the kernel parameter (about 9 KB; CUDA >= 12.1 allows 32 KB): the
// schedule then lives in the constant bank, indexed with uniform registers, so that every
// test on it is a uniform branch (no convergence barriers, no shared-memory latency).
struct ScanParams {
  const float* packed = nullptr;   // [n_ct][dim][CW][TILE_C]
  const float* qpacked = nullptr;  // [n_qt][dim][QW][TILE_Q]
  const float* s_true = nullptr;   // [n_qt*TILE_Q], NaN padded
  const uint8_t* code_host = nullptr;  // [dim] schedule codes (HOST pointer; copied into `code` at launch)
  int32_t* counts = nullptr;       // [n_q] (+=) or nullptr
  float* scores = nullptr;         // [n_q][n_rows] or nullptr
  // bound-and-refine form (RotatE): approximate element arithmetic, pairs whose approximate
  // score is within rel_eps * |score| of s_true go to the near-tie list (regions of 128 queries)
  unsigned long long* amb_count = nullptr;  // [ceil(n_q / 128)] or nullptr (exact scan)
  int2* amb_pairs = nullptr;                // [regions][amb_cap]
  unsigned long long amb_cap = 0;
  float rel_eps = 0.f;
  float abs_eps = 0.f;   // flushed subnormal terms: dim * 1.1e-19
  // top-k collect form (kge_topk_side): s_true holds a per-query THRESHOLD; every candidate whose
  // exact score is not below it is appended to the query's list as (score bits, global id)
  int2* col_buf = nullptr;        // [n_q][col_cap] or nullptr
  unsigned* col_count = nullptr;  // [n_q] fill counts (unused when col_dense)
  unsigned long long col_cap = 0;
  long long col_id_base = 0;      // global id of candidate row 0 of this launch
  int col_dense = 0;              // 1: slot = row index (first chunk: everything is collected)
  int dim = 0;
  int64_t n_q = 0;
  int64_t n_rows = 0;
  int64_t n_ct = 0;
  int64_t n_qt = 0;
  // filled by launch_scan from code_host
  uint32_t mask[SCAN_MAX_DIM / SCAN_KC];  // per stage: bit kk set <=> position needs the slow path
  uint8_t code[SCAN_MAX_DIM];
};
static_assert(std::is_trivially_copyable<ScanParams>::value, "ScanParams is a kernel parameter");

// Calls f(std::integral_constant<int, EL>{}, std::bool_constant<CASC>{}) for the element kind `el`
// and the schedule's cascade flag, and returns what f returns.  Only the kinds reduced by the cascade
// sum (RED_SUM) have a CASC = true form; the norm kinds are always called with CASC = false.  An
// unknown kind gives cudaErrorInvalidValue.
template <class F>
cudaError_t dispatch_elem(int el, bool cascade, F&& f) {
  auto with = [&](auto kind) -> cudaError_t {
    if constexpr (ElemTraits<decltype(kind)::value>::RED == RED_SUM)
      if (cascade) return f(kind, std::true_type{});
    return f(kind, std::false_type{});
  };
  switch (el) {
    case EL_DOT1: return with(std::integral_constant<int, EL_DOT1>{});
    case EL_DOT2: return with(std::integral_constant<int, EL_DOT2>{});
    case EL_DOT3: return with(std::integral_constant<int, EL_DOT3>{});
    case EL_ROT: return with(std::integral_constant<int, EL_ROT>{});
    case EL_DOT_MID: return with(std::integral_constant<int, EL_DOT_MID>{});
    case EL_TL1_TAIL: return with(std::integral_constant<int, EL_TL1_TAIL>{});
    case EL_TL1_HEAD: return with(std::integral_constant<int, EL_TL1_HEAD>{});
    case EL_TL2_TAIL: return with(std::integral_constant<int, EL_TL2_TAIL>{});
    case EL_TL2_HEAD: return with(std::integral_constant<int, EL_TL2_HEAD>{});
    case EL_L1_TAIL: return with(std::integral_constant<int, EL_L1_TAIL>{});
    case EL_L1_HEAD: return with(std::integral_constant<int, EL_L1_HEAD>{});
    case EL_L2_TAIL: return with(std::integral_constant<int, EL_L2_TAIL>{});
    case EL_L2_HEAD: return with(std::integral_constant<int, EL_L2_HEAD>{});
    default: return cudaErrorInvalidValue;
  }
}

// dense scan: counts[q] += #{c < n_rows : score(q,c) >= s_true[q]}  (or writes scores)
// approx = true (EL_ROT only): the bound-and-refine form above; p.amb_* and p.rel_eps must be set
cudaError_t launch_scan(int el, bool cascade, const ScanParams& p, cudaStream_t stream,
                        bool approx = false);

// packed[ct][pos][plane][TILE_C] <- ent_plane[row][perm[pos]]
cudaError_t launch_pack_table(const float* ent0, const float* ent1, int planes, int64_t n_rows,
                              int dim, const int32_t* inv_perm, float* packed,
                              cudaStream_t stream);

cudaError_t launch_gather_rows(const float* ent0, const float* ent1, int planes, int64_t ent_lo,
                               int64_t n_rows, int dim, const int64_t* idx, int64_t n,
                               float* out, cudaStream_t stream);

// qplain[i][plane][dim] from the gathered head/tail rows and the relation tables
cudaError_t launch_prep_queries(int model, int side, int dim, int64_t n, const float* hrows,
                                const float* trows, const float* rel0, const float* rel1,
                                const int64_t* r_idx, float* qplain, cudaStream_t stream);

// qpacked[qt][pos][plane][TILE_Q] <- qplain[i][plane][perm[pos]] (zero padded)
cudaError_t launch_pack_queries(const float* qplain, int qw, int dim, int64_t n,
                                const int32_t* perm, float* qpacked, cudaStream_t stream);

cudaError_t launch_fill_f32(float* dst, float value, int64_t n, cudaStream_t stream);

// s_true[i] = score(query i, rows[i])   (rows = [n][CW][dim])
cudaError_t launch_true_scores(int el, bool cascade, int dim, int64_t n, const float* qplain,
                               const float* rows, const int32_t* perm, const uint8_t* code,
                               float* s_true, cudaStream_t stream);

// filt_sub[q] += [s(q,c) >= s_true[q]] - [s_true[q] == -inf] for every CSR entry c of q that
// lies in [ent_lo, ent_lo + n_rows)
cudaError_t launch_filter(int el, bool cascade, int dim, int64_t n, int64_t n_filt,
                          const float* qplain,
                          const float* ent0, const float* ent1, int64_t ent_lo, int64_t n_rows,
                          const int64_t* offs, const int64_t* ids, const int32_t* qid, const int32_t* perm,
                          const uint8_t* code, const float* s_true, int32_t* filt_sub,
                          cudaStream_t stream);

cudaError_t launch_finalize(const int32_t* raw, const int32_t* sub, int64_t n, int64_t* ranks,
                            int64_t* filt_ranks, cudaStream_t stream);

// out[row][k] = TransH projection of ent[row] on the hyperplane of normal w (reduce.cuh: transh_project_elem)
cudaError_t launch_transh_project(const float* ent, const float* w, int64_t n_rows, int dim, float* out,
                                  cudaStream_t stream);
// s[row] = (ent_proj[row] * ent[row]).sum() in ATen's order: TransD's per-entity scalar
cudaError_t launch_transd_entity_scalars(const float* ent, const float* ent_proj, int64_t n_rows, int ent_dim,
                                         float* s, cudaStream_t stream);
// out[row][j] = TransD projection of ent[row] (row stride ent_dim) under one relation, j < rel_dim
// (reduce.cuh: transd_project_elem)
cudaError_t launch_transd_project(const float* ent, int ent_dim, const float* s, const float* rel_proj_row,
                                  int64_t n_rows, int rel_dim, float* out, cudaStream_t stream);

// ---- top-k selection over collected candidates (topk.cu) ----
// best[q][k] sorted 64-bit keys (score order, then smaller id first; 0 = empty slot).
// Merges the `count[q]` (or `dense_count`) entries of col_buf[q] into best[q], masking ids listed in
// the query's sorted CSR row with -inf (filter_scores with true_idx = None, utils/modeling.py:91-102),
// and writes the new threshold thr[q] (the k-th best score, -inf while fewer than k are held).
cudaError_t launch_topk_merge(unsigned long long* best, int k, const int2* col_buf,
                              const unsigned* col_count, unsigned long long col_cap, long long dense_count,
                              const int64_t* mask_offs, const int64_t* mask_ids, float* thr, int64_t n_q,
                              cudaStream_t stream);
// pred[q][j], scores[q][j] from the keys
cudaError_t launch_topk_finish(const unsigned long long* best, int k, int64_t n_q, int64_t* pred,
                               float* scores, cudaStream_t stream);
constexpr int TOPK_MAX_K = 1024;
constexpr int TOPK_MAX_LISTS = 64;
// pred[q][0..k) / scores[q][0..k): the k best entries of the union of n_lists sorted lists
// pred_in / scores_in [n_lists][n][k_in] (same key order as above; pred < 0 marks an empty slot)
cudaError_t launch_topk_lists_merge(const int64_t* pred_in, const float* scores_in, int n_lists, int64_t n,
                                    int k_in, int k, int64_t* pred, float* scores, cudaStream_t stream);

// ---- dense side paths (dense.cu) ----
// scores[i][c] = ((h_i^T M_c) * t_i).sum()   RESCAL relation case, bilinear.py:115-121
cudaError_t launch_rescal_rel_scores(const float* hrows, const float* trows, const float* rel_mat, int dim,
                                     int64_t n, int64_t n_rel, float* scores, cudaStream_t stream);
// scores[i][c] = -||(P_c(h_i) + r_c) - P_c(t_i)||^2   TransH relation case, interfaces.py:261-272
cudaError_t launch_transh_rel_scores(const float* hrows, const float* trows, const float* rel,
                                     const float* norm_vect, int dim, int64_t n, int64_t n_rel, float* scores,
                                     cudaStream_t stream);
// scores[i][c] = -||(P_c(h_i) + r_c) - P_c(t_i)||^2   TransD relation case, P_c from the first dim
// coordinates of the rows and their scalars hs / ts
cudaError_t launch_transd_rel_scores(const float* hrows, const float* hs, const float* trows, const float* ts,
                                     const float* rel, const float* rel_proj, int dim, int64_t n, int64_t n_rel,
                                     float* scores, cudaStream_t stream);
cudaError_t launch_rank_dense(const float* scores, int64_t n, int64_t n_c, const int64_t* true_idx,
                              const float* true_score_in, const int64_t* offs, const int64_t* ids,
                              int32_t* raw_count, int32_t* filt_sub, float* true_score_out, cudaStream_t stream);
cudaError_t launch_dense_to_pairs(const float* scores, int64_t n, int64_t n_c, int2* pairs, cudaStream_t stream);

// ---- relation co-occurrence of the data-redundancy analysis (redundancy.cu) ----
// counts[r_a * n_rel + r_b] += 1 for every key r_a of a left segment and r_b of the right segment with the
// same (h, t) pair, or (t, h) when flip; upper: only r_a < r_b
cudaError_t launch_cooccurrence(const int64_t* lkeys, const int64_t* loffs, const int64_t* lpairs, int64_t n_left,
                                const int64_t* rkeys, const int64_t* roffs, const int64_t* rpairs, int64_t n_right,
                                int64_t n_ent, int64_t n_rel, bool flip, bool upper, unsigned long long* counts,
                                cudaStream_t stream);

}  // namespace kge
