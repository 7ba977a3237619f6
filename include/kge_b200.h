/*
 * kge_b200.h -- C ABI of the H100-native (sm_90a) KG-embedding scoring / link-prediction
 * ranking engine (libkge_b200.so).
 *
 * The reference (torchkge @ 3adb934, v0.17.7) has no FFI of its own: its hot path is
 * Python over ATen.  Every entry point below therefore names the reference Python
 * symbol (file:line in torchkge 0.17.7) whose tensor-op body it replaces; the
 * Python shim in torchkge_b200/ keeps the reference's class/method signatures and
 * calls these through ctypes (see INTEGRATION.md for the binding).
 *
 * Conventions
 *   - plain pointers and sizes only; no torch types.  All `const float*`/`int64_t*`
 *     pointers are DEVICE pointers unless the name ends in `_host`.
 *   - the caller owns every buffer (the shim allocates them as torch tensors);
 *     the library allocates nothing persistent.
 *   - every call enqueues work on `stream` (a cudaStream_t passed as void*) and
 *     returns without synchronising.
 *   - return value: 0 = ok, nonzero = error code (KGE_ERR_*); kge_last_error()
 *     returns a thread-local message.  Nothing throws or aborts.
 *   - all embeddings are fp32 row-major with leading dimension = dim; all entity /
 *     relation indices are int64; rank counters are int32 on device and widened to
 *     int64 by kge_finalize_ranks().
 *
 * Arithmetic contract ("ATen order"): for one (query, candidate) pair the score is
 * evaluated with exactly the fp32 operation sequence torchkge executes on its CPU
 * path through ATen 2.11 (separately rounded mul/add, 8-lane vector accumulation,
 * cascade summation, sqrt-then-square for L2) -- see DESIGN.md "Reduction
 * schedules".  The sequence depends only on (model, side, dim), never on tile /
 * thread / shard position, so equal inputs give bit-equal scores everywhere and
 * ranks equal the reference's CPU ranks bit for bit.
 */
#ifndef KGE_B200_H
#define KGE_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define KGE_ABI_VERSION 11

/* error codes */
#define KGE_OK 0
#define KGE_ERR_ARG 1     /* bad argument (null pointer, unsupported dim, ...) */
#define KGE_ERR_CUDA 2    /* a CUDA runtime call failed; see kge_last_error() */
#define KGE_ERR_UNSUPPORTED 3

/* Scoring models on the path (SURVEY.md section 8a rows a3-a6, a14). */
typedef enum {
  KGE_TRANSE_L1 = 0, /* torchkge/models/translation.py:18  + utils/dissimilarities.py:11 */
  KGE_TRANSE_L2 = 1, /* torchkge/models/translation.py:18  + utils/dissimilarities.py:19 */
  KGE_DISTMULT = 2,  /* torchkge/models/bilinear.py:146 */
  KGE_RESCAL = 3,    /* torchkge/models/bilinear.py:14 */
  KGE_COMPLEX = 4,   /* torchkge/models/bilinear.py:414 */
  KGE_ROTATE = 5,    /* not in the reference; oracle/rotate restatement (Sun et al. 2019) */
  KGE_TORUSE_L1 = 6, /* torchkge/models/translation.py:655 + utils/dissimilarities.py:28-34 (torus_L1);
                        link-prediction side only (kge_rank_side / kge_score_all), tables already
                        reduced to their fractional parts (TorusEModel.normalize_parameters) */
  KGE_TORUSE_L2 = 7, /* same + utils/dissimilarities.py:37-43 (torus_L2); torus_eL2 (cosine) is not
                        on the path */
  KGE_ANALOGY = 8    /* torchkge/models/bilinear.py:559-763, scalar_dim == complex_dim == dim: THREE planes
                        per row (scalar, real, imaginary), see "three-plane tables" below */
} kge_model_t;

/* Three-plane tables (KGE_ANALOGY).  Every entry point takes at most two pointers per table
 * (ent0 / ent1, rel0 / rel1, hrows / trows rows of [planes][dim]).  For a three-plane model the planes
 * of a table must be EQUALLY SPACED in memory -- e.g. one [3][n_rows][dim] array, or row ranges of
 * one -- and the caller passes planes 0 and 1: the library reads plane 2 at ent1 + (ent1 - ent0)
 * (likewise rel1 + (rel1 - rel0), and for gradient tables).  No signature changes with the number
 * of planes. */

/* Which element of the triple is being completed. */
typedef enum {
  KGE_SIDE_TAIL = 0, /* (h, r, ?)  evaluation.py:292 */
  KGE_SIDE_HEAD = 1, /* (?, r, t)  evaluation.py:297 */
  KGE_SIDE_REL = 2   /* (h, ?, t)  RelationPredictionEvaluator, evaluation.py:94-97: the candidate
                        table (packed / ent0 / ent1) is the RELATION table (rel_emb; re_/im_rel_emb),
                        rel0 / rel1 / r_idx are unused, true_rows is required.  TransE L1/L2, DistMult,
                        ComplEx, Analogy (RESCAL's batched matmul and RotatE are not on this path). */
} kge_side_t;

/* Geometry of the packed layouts, fixed at build time; exported so that callers can
 * size buffers.  A "candidate tile" is KGE_TILE_C consecutive entity rows, a "query
 * tile" is KGE_TILE_Q consecutive queries. */
#define KGE_TILE_C 128
#define KGE_TILE_Q 64

int kge_abi_version(void);
const char* kge_last_error(void);

/* Number of fp32 planes per entity row / per query for a model:
 * candidates: 1 (TransE, DistMult, RESCAL), 2 (ComplEx, RotatE: re, im) or 3 (Analogy: sc, re, im);
 * queries: 1, or 2 for TransE head side (r and t stay separate, interfaces.py:256-260)
 * and for ComplEx / RotatE, 3 for Analogy. */
int kge_cand_planes(int model);
int kge_query_planes(int model, int side);

/* ---- reduction schedule (host only; no GPU needed) ------------------------------
 * Fills perm_host[dim] (schedule position -> original embedding index) and
 * code_host[dim] (combine micro-ops executed after each position) for the reduction
 * the reference performs for `model`: sequential (L1 norm), 8-lane norm (L2), or
 * ATen's cascade sum (bilinear models / RotatE).  Exposed for CPU tests, which
 * replay the schedule in numpy and compare with ATen bit for bit. */
int kge_build_schedule(int model, int dim, int32_t* perm_host, uint8_t* code_host);
/* Depth of that reduction tree: the most rounded additions any term passes through (-1 if the
 * model / dim is unsupported).  The tensor-core path's error bound uses it (host only). */
int kge_schedule_depth(int model, int dim);

/* ---- table packing ---------------------------------------------------------------
 * Re-lays an entity table shard (rows [0, n_rows) of ent0 / ent1, each row-major
 * [n_rows][dim]; ent1 only for 2-plane models) into the scan layout
 *   packed[ctile][pos][plane][KGE_TILE_C]      (pos = schedule position, 0..dim-1)
 * so that one pipeline stage of the scan is a single contiguous bulk copy.
 * Replaces the zero-copy `expand` of ent_emb.weight in inference_prepare_candidates
 * (translation.py:105-125, bilinear.py:123-143, 247-267, 530-556). */
/* ---- tensor-core operand image of a table shard (optional, see kge_rank_args_t.flags) ----
 * For models whose score is a dot product or a squared L2 distance (DistMult, RESCAL, ComplEx, Analogy,
 * TransE-L2) the dense scan can run as a split GEMM (x = hi + lo in bf16 or fp16, three MMAs per
 * fp32 product) on the tensor cores that decides
 * every (query, candidate) pair whose approximate score differs from the true score by more
 * than a rigorous error bound, the remaining near-ties being re-scored exactly -- ranks are
 * unchanged.  kge_tc_pack_table writes the operand image that path streams:
 * [hi/lo half-precision planes in swizzled shared-memory order (64-byte swizzle spans by default,
 * see kge_tc_configure) | per-row norm bounds and squared norms | 256 bytes of per-image facts
 * (scale, maxima) established on the device].
 * kge_tc_packed_bytes returns 0 for models without such a path (TransE-L1, RotatE). */
size_t kge_tc_packed_bytes(int model, int64_t n_rows, int dim);
/* Tuning / test hook of the tensor-core scan (process-wide; defaults also settable through the
 * environment: KGE_TC_BK, KGE_TC_RESIDENT, KGE_TC_GROUP, KGE_TC_MAX_CTAS).  bk = bf16 per k-block
 * (32: 64-byte swizzle, query-tile image resident in shared memory when k <= 224; 64: 128-byte
 * swizzle, both operands streamed); ct_group = candidate tiles per work unit (0 = automatic);
 * max_ctas = grid limit (0 = one CTA per SM); fp16 = operand format of the split (0: bf16, residual
 * 2^-16 |x|; 1: fp16 with a per-image power-of-two pre-scale, residual 2^-22 |x|, i.e. a narrower
 * near-tie band; KGE_TC_FP16).  Negative arguments keep the current value.
 * Images packed under one (bk, fp16) must be scanned under the same.  Results never depend on it. */
int kge_tc_configure(int bk, int resident, int ct_group, int max_ctas, int fp16);
/* (host only) identifies the operand-image layout kge_tc_configure currently selects (k-block width
 * and operand format): an image may only be scanned under the layout it was packed under. */
int kge_tc_layout_id(void);
/* kge_tc_pack_table for callers that KEEP the image between evaluations: `guard` = 4 device uint64
 * (zero-initialised once, owned by the caller together with tc_packed).  The call computes a 128-bit
 * content checksum of the table (one read of the table at HBM speed) and rebuilds the image only
 * when it differs from the checksum recorded at the last rebuild -- in-place weight updates of any
 * kind (optimizer steps, `.data` edits) are therefore always picked up.  guard = NULL: always rebuild. */
int kge_tc_pack_table_cached(int model, const float* ent0, const float* ent1, int64_t n_rows, int dim,
                             void* tc_packed, uint64_t* guard, void* stream);
/* (host only) The constants of the rigorous error bound the tensor-core scan uses for `model` at
 * `dim` under the current operand format (csrc/tc.h: tc_gamma, tc_gamma2, tc_gamma_p):
 *   dot models : |s_tc - s_ref| <= gamma |a| |b| + gamma_p P(a) P(b)
 *   TransE-L2  : |s_tc - s_ref| <= 2 gamma |a| |b| + 2 gamma_p P(a) P(b) + gamma2 (|a| + |b|)^2
 * |a|, |b|: per-row norm bounds (inflated by TcMeta::kappa under fp16); P(x) = sqrt(sum_i |x_{<=16 i}|^2),
 * the running-magnitude factor of the accumulation inside the tensor core.  Exposed so that the tests
 * check the measured error against exactly what the kernel assumes. */
int kge_tc_bound_constants(int model, int dim, float* gamma, float* gamma2, float* gamma_p, int* fp16);
int kge_tc_pack_table(int model, const float* ent0, const float* ent1, int64_t n_rows, int dim,
                      void* tc_packed, void* stream);

size_t kge_packed_table_floats(int model, int64_t n_rows, int dim);
int kge_pack_table(int model, const float* ent0, const float* ent1, int64_t n_rows, int dim,
                   float* packed, void* stream);

/* ---- query rows --------------------------------------------------------------------
 * out[i][plane][dim] = ent_plane[idx[i] - ent_lo]  if ent_lo <= idx[i] < ent_lo+n_rows
 *                      else 0                                   (i < n)
 * (the Embedding lookups of inference_prepare_candidates).  With a range-partitioned
 * table each rank calls this on its shard and the shim sum-all-reduces `out`. */
int kge_gather_rows(int model, const float* ent0, const float* ent1, int64_t ent_lo,
                    int64_t n_rows, int dim, const int64_t* idx, int64_t n, float* out,
                    void* stream);

/* ---- link-prediction ranking: the hot path ---------------------------------------
 * One call ranks n test triples on one side against the entity rows
 * [ent_lo, ent_lo + n_rows) held by this GPU.  It fuses, without ever writing an
 * (n, n_ent) score matrix:
 *   inference_scoring_function   (interfaces.py:240-260, bilinear.py:98-121,
 *                                 224-245, 501-528)
 *   filter_scores / get_true_targets (utils/modeling.py:53-102)
 *   get_rank                     (utils/operations.py:37-61)
 * Results are ADDED into the int32 counters
 *   raw_count[i]  += #{c in shard : s(i,c) >= s_true(i)}
 *   filt_sub[i]   += #{c in shard, c in F(i)\{true} : s(i,c) >= s_true(i) and s_true(i) > -inf}
 * so that rank_raw = sum over shards of raw_count and rank_filt = rank_raw - sum of
 * filt_sub (one sum-all-reduce when sharded).
 */
typedef struct {
  int32_t model; /* kge_model_t */
  int32_t side;  /* kge_side_t */
  int32_t dim;
  int32_t flags;  /* KGE_FLAG_* */
  int64_t n;      /* triples in this call */
  int64_t n_ent;  /* global number of entities */
  int64_t ent_lo; /* first global entity id held in `packed` / ent0 / ent1 */
  int64_t n_rows; /* rows held */
  const float* packed; /* kge_pack_table output for this shard (may be NULL when the tensor-core
                          scan is used: KGE_FLAG_TENSOR_CORE and a model that has one) */
  const float* ent0;   /* row-major shard (used for the sparse filter pass) */
  const float* ent1;   /* second plane or NULL */
  const float* rel0;   /* relation table: rel_emb / re_rel_emb / rel_mat / phases */
  const float* rel1;   /* im_rel_emb or NULL */
  const float* hrows;  /* [n][cand_planes][dim] rows of the heads (kge_gather_rows) */
  const float* trows;  /* [n][cand_planes][dim] rows of the tails */
  const int64_t* r_idx;    /* [n] relation ids; NULL: rel0/rel1 hold one row per triple */
  const int64_t* true_idx; /* [n] global id of the true entity on this side */
  /* CSR of the filter sets, true entity already removed, quirks of
   * get_true_targets already applied by the shim: */
  const int64_t* filt_offs; /* [n+1] or NULL (no filtering) */
  const int64_t* filt_ids;  /* [n_filt] global entity ids */
  int64_t n_filt;           /* = filt_offs[n], known to the host */
  int32_t* raw_count;       /* [n] += */
  int32_t* filt_sub;        /* [n] += */
  float* true_score;        /* [n] out (optional, may be NULL): s_true */
  void* workspace;          /* kge_rank_workspace_bytes() bytes, 256-B aligned */
  size_t workspace_bytes;
  void* stream;
  const void* tc_packed;    /* kge_tc_pack_table output (required with KGE_FLAG_TENSOR_CORE) */
  uint64_t* tc_stats;       /* optional device out [2]: near-tie pairs found, list capacity;
                               found > capacity means the list overflowed and the counters of
                               this call are INVALID: redo the call without the flag */
  float* tc_dump;           /* debug / tests: if set, the tensor-core pass writes its approximate
                               scores [n][n_rows] here and counts nothing */
  const float* true_rows;   /* [n][cand_planes][dim] rows of the true candidates; NULL: trows (tail
                               side) / hrows (head side).  Required for KGE_SIDE_REL. */
  const float* true_score_in; /* [n] or NULL: use these true scores instead of scoring true_rows
                               (undirected relation prediction ranks the swapped (t, ?, h) scores
                               against the directed true score, evaluation.py:99-107) */
  const int32_t* filt_qid;  /* [n_filt] or NULL: the triple (row of the CSR) every filter entry belongs to;
                               saves the filter pass a binary search in filt_offs per entry */
} kge_rank_args_t;

#define KGE_FLAG_TENSOR_CORE 1 /* use the tensor-core bound-and-refine scan when the model has one */
#define KGE_FLAG_APPROX_SCAN 2 /* RotatE: bound-and-refine on the fp32 pipes -- approximate element
                                  arithmetic (FMA + MUFU.SQRT, two-level sums) decides every pair
                                  outside a rigorous relative error band around the true score, the
                                  rest is re-scored exactly; ranks unchanged.  tc_stats as above. */

/* n_rows / flags only matter for the tensor-core path (near-tie list capacity). */
size_t kge_rank_workspace_bytes(int model, int side, int dim, int64_t n, int64_t n_rows, int flags);
int kge_rank_side(const kge_rank_args_t* args);
/* Only the sparse filter pass of kge_rank_side, for callers that enqueue the dense scan first
 * (filt_offs = NULL) and build the filter CSR on the host while it runs: `args` must be the
 * arguments of that earlier kge_rank_side call -- same workspace, still intact -- now with
 * filt_offs / filt_ids / n_filt / filt_sub set. */
int kge_filter_side(const kge_rank_args_t* args);

/* ranks[i] = raw_count[i] (int32 -> int64); filt_ranks[i] = raw_count[i] - filt_sub[i]
 * (evaluation.py:294-300 store int64). */
int kge_finalize_ranks(const int32_t* raw_count, const int32_t* filt_sub, int64_t n,
                       int64_t* ranks, int64_t* filt_ranks, void* stream);

/* ---- dense scores (API parity, not the hot path) ----------------------------------
 * scores[i][c] for all c in the shard, row-major (n, n_rows): what
 * inference_scoring_function returns.  Same arithmetic as kge_rank_side. */
typedef struct {
  int32_t model, side, dim, reserved0;
  int64_t n;
  int64_t n_rows;
  const float* packed;
  const float* rel0;
  const float* rel1;
  const float* hrows;
  const float* trows;
  const int64_t* r_idx; /* NULL: rel0/rel1 hold one row per triple (already gathered) */
  float* scores; /* [n][n_rows] */
  void* workspace;
  size_t workspace_bytes;
  void* stream;
} kge_score_all_args_t;
int kge_score_all(const kge_score_all_args_t* args);

/* ---- top-k inference (EntityInference / RelationInference, torchkge/inference.py:78-250) ------
 * pred[i][0..k) / scores[i][0..k): the k best candidates of query i and their exact (ATen-order)
 * scores, best first -- what the reference obtains from inference_scoring_function, filter_scores
 * (true_idx = None: every listed candidate masked with -inf, utils/modeling.py:91-102) and
 * sort(descending=True)[:, :k] -- without an (n, n_rows) score matrix: the dense scan runs in a
 * collect mode that writes out only candidates not below the query's current k-th best, a chunk of
 * candidate rows at a time, merged into a per-query sorted list after every chunk.  NaN ranks above
 * everything (as in torch's sort); exact ties are ordered by ascending candidate id.
 * With a range-partitioned table, `packed` holds the rows [ent_lo, ent_lo + n_rows): pred holds
 * global ids (ent_lo + row), the mask CSR lists global ids, and kge_topk_merge combines the lists of
 * the shards into the unsharded result. */
typedef struct {
  int32_t model, side, dim, k;   /* 1 <= k <= 1024, k <= n_rows */
  int64_t n;                     /* queries */
  int64_t n_rows;                /* candidates (rows of the packed table) */
  const float* packed;           /* kge_pack_table output of the candidate table */
  const float* rel0;
  const float* rel1;
  const float* hrows;
  const float* trows;
  const int64_t* r_idx;          /* as in kge_score_all_args_t */
  const int64_t* mask_offs;      /* [n+1] CSR of candidates to mask with -inf, or NULL */
  const int64_t* mask_ids;       /* candidate ids, ASCENDING within each row */
  int64_t* pred;                 /* [n][k] out */
  float* scores;                 /* [n][k] out */
  void* workspace;               /* kge_topk_workspace_bytes() bytes, 256-B aligned */
  size_t workspace_bytes;
  void* stream;
  int64_t ent_lo;                /* global id of row 0 of `packed` (0: unsharded); ent_lo + n_rows < 2^31 */
} kge_topk_args_t;
size_t kge_topk_workspace_bytes(int model, int side, int dim, int64_t n, int64_t n_rows, int k);
int kge_topk_side(const kge_topk_args_t* args);
/* pred[i][0..k) / scores[i][0..k): the k best entries of the union of n_lists lists
 * pred_in / scores_in [n_lists][n][k_in], each sorted best first as kge_topk_side returns them, pred = -1
 * marking an empty slot (at the end of a list).  Same order as kge_topk_side: score bits (NaN on top,
 * +0.0 above -0.0), then ascending id; empty slots last, output as (-1, -inf).  Ids must be unique
 * across the lists (disjoint shards), which makes the result that of one unsharded call.
 * 1 <= n_lists <= 64, 1 <= k, k_in <= 1024; anything else returns KGE_ERR_ARG. */
int kge_topk_merge(const int64_t* pred_in, const float* scores_in, int n_lists, int64_t n, int k_in, int k,
                   int64_t* pred, float* scores, void* stream);

/* ---- dense side paths -----------------------------------------------------------------------
 * RESCAL relation prediction (models/bilinear.py:115-121): the candidates are the relation matrices,
 * scores[i][c] = ((h_i^T M_c) * t_i).sum() -- batched matmul in the reference's (oneMKL) summation
 * order, then the ATen cascade sum.  hrows / trows: [n][dim] rows of the heads / tails, rel_mat:
 * [n_rel][dim*dim], scores: [n][n_rel] out.  The matrix is small (n_rel columns) and is what
 * kge_rank_dense / kge_topk_dense consume. */
int kge_rescal_rel_scores(const float* hrows, const float* trows, const float* rel_mat, int dim, int64_t n,
                          int64_t n_rel, float* scores, void* stream);
/* TransH relation prediction (models/interfaces.py:261-272 with the projections of
 * models/translation.py:253-254): scores[i][c] = -||(P_c(h_i) + r_c) - P_c(t_i)||^2, where
 * P_c(e) = e - (e . w_c) w_c is computed as kge_transh_project computes it and the norm is summed in
 * ATen's L2-norm order.  hrows / trows: [n][dim] raw entity rows, rel / norm_vect: [n_rel][dim]
 * (rel_emb.weight, norm_vect.weight), scores: [n][n_rel] out, for kge_rank_dense / kge_topk_dense.
 * dim <= 8192. */
int kge_transh_rel_scores(const float* hrows, const float* trows, const float* rel, const float* norm_vect,
                          int dim, int64_t n, int64_t n_rel, float* scores, void* stream);
/* TransD relation prediction (models/interfaces.py:261-272 with the projections of
 * models/translation.py:645-646): scores[i][c] = -||(P_c(h_i) + r_c) - P_c(t_i)||^2, where
 * P_c(e)[j] = fl(fl(s_e * rel_proj[c][j]) + e[j]) as kge_transd_project computes it and the norm is summed in
 * ATen's L2-norm order.  hrows / trows: [n][rel_dim] the first rel_dim coordinates of the raw ent_emb rows,
 * hs / ts: [n] their scalars (kge_transd_entity_scalars), rel / rel_proj: [n_rel][rel_dim] (rel_emb.weight,
 * rel_proj_vect.weight), scores: [n][n_rel] out, for kge_rank_dense / kge_topk_dense.  rel_dim <= 8192. */
int kge_transd_rel_scores(const float* hrows, const float* hs, const float* trows, const float* ts, const float* rel,
                          const float* rel_proj, int rel_dim, int64_t n, int64_t n_rel, float* scores, void* stream);
/* get_rank + filter_scores (utils/operations.py:37-61, utils/modeling.py:91-102) on a dense (n, n_cand)
 * score matrix, counters ADDED INTO as by kge_rank_side: raw_count[i] += #{c : s >= s_true};
 * filt_sub[i] += listed candidates with s >= s_true (minus the -inf quirk).  s_true = true_score_in[i]
 * if given (undirected second pass) else scores[i][true_idx[i]]; true_score (optional) receives it. */
int kge_rank_dense(const float* scores, int64_t n, int64_t n_cand, const int64_t* true_idx,
                   const float* true_score_in, const int64_t* filt_offs, const int64_t* filt_ids,
                   int32_t* raw_count, int32_t* filt_sub, float* true_score, void* stream);
/* the k best columns of every row of a dense matrix, masked candidates set to -inf (same ordering
 * rules as kge_topk_side) */
size_t kge_topk_dense_workspace_bytes(int64_t n, int64_t n_cand, int k);
int kge_topk_dense(const float* scores, int64_t n, int64_t n_cand, int k, const int64_t* mask_offs,
                   const int64_t* mask_ids, int64_t* pred, float* out_scores, void* workspace,
                   size_t workspace_bytes, void* stream);

/* ---- training side ----------------------------------------------------------------------
 * Tables as in ModelSpec order: ent0/ent1 entity planes (n_ent, dim), rel0/rel1 relation
 * planes (n_rel, dim) -- RESCAL: rel0 = rel_mat (n_rel, dim*dim); RotatE: (cos, sin) of the
 * phases.  Gradient tables have the same shapes, are zero-initialised by the caller and are
 * accumulated into with atomics (dense gradients, as nn.Embedding produces). */
typedef struct {
  int32_t model, dim;
  const float* ent0; const float* ent1; const float* rel0; const float* rel1;
} kge_tables_t;
typedef struct {
  float* ent0; float* ent1; float* rel0; float* rel1;
} kge_grads_t;

/* TransH's projected entity table for one relation (models/translation.py:270-284, evaluate_projections):
 * out[e][k] = fl(ent[e][k] - fl(nc_e * w[k])), nc_e = (ent[e] * w).sum() summed in ATen's inner-dimension
 * order.  ent: [n_rows][dim] raw ent_emb.weight, norm_row: [dim] raw norm_vect.weight row, out: [n_rows][dim]
 * (caller-provided).  The result feeds kge_pack_table / kge_tc_pack_table and kge_rank_side /
 * kge_topk_side as a KGE_TRANSE_L2 table.  dim <= 8192. */
int kge_transh_project(const float* ent, const float* norm_row, int64_t n_rows, int dim, float* out,
                       void* stream);
/* TransD's per-entity scalar (models/translation.py:645, evaluate_projectionss):
 * s[e] = (ent_proj[e] * ent[e]).sum() summed over ent_dim in ATen's inner-dimension order.  ent / ent_proj:
 * [n_rows][ent_dim] raw ent_emb.weight / ent_proj_vect.weight, s: [n_rows] out.  It does not depend on the
 * relation: one call serves every kge_transd_project of an evaluation.  ent_dim <= 8192. */
int kge_transd_entity_scalars(const float* ent, const float* ent_proj, int64_t n_rows, int ent_dim, float* s,
                              void* stream);
/* TransD's projected entity table for one relation (models/translation.py:646):
 * out[e][j] = fl(fl(s[e] * rel_proj_row[j]) + ent[e][j]) for j < rel_dim, two roundings as in the reference.
 * ent: [n_rows][ent_dim] raw ent_emb.weight (read with row stride ent_dim), s: [n_rows] from
 * kge_transd_entity_scalars, rel_proj_row: [rel_dim] raw rel_proj_vect.weight row, out: [n_rows][rel_dim]
 * (caller-provided).  The result feeds the scans as a KGE_TRANSE_L2 table of width rel_dim.
 * rel_dim <= ent_dim <= 8192. */
int kge_transd_project(const float* ent, int ent_dim, const float* s, const float* rel_proj_row, int64_t n_rows,
                       int rel_dim, float* out, void* stream);

/* Model.scoring_function (models/translation.py:69-81, models/bilinear.py:60-71, 188-199,
 * 460-473): scores[i] of triple (h[i], r[i], t[i]); TransE / DistMult / RESCAL L2-normalise
 * the gathered entity rows first (eps 1e-12). */
int kge_score_triples_fwd(const kge_tables_t* tb, const int64_t* h, const int64_t* t,
                          const int64_t* r, int64_t n, float* scores, void* stream);
/* accumulates d(sum_i grad_scores[i] * scores[i]) / d(tables) into g */
int kge_score_triples_bwd(const kge_tables_t* tb, const kge_grads_t* g, const int64_t* h,
                          const int64_t* t, const int64_t* r, int64_t n, const float* grad_scores,
                          void* stream);
/* TransH's scoring_function (models/translation.py:183-202): scores[i] = -||P(h~) + r - P(t~)||^2 with h~,
 * t~ and the relation's normal vector w~ L2-normalised (eps 1e-12) and P(v) = v - (v . w~) w~.  Its own
 * tables (ent_emb.weight, rel_emb.weight, norm_vect.weight, each [rows][dim]) rather than a kge_tables_t. */
int kge_transh_score_triples_fwd(const float* ent, const float* rel, const float* norm_vect, int dim,
                                 const int64_t* h, const int64_t* t, const int64_t* r, int64_t n, float* scores,
                                 void* stream);
/* accumulates d(sum_i grad_scores[i] * scores[i]) / d(tables) into the three gradient tables */
int kge_transh_score_triples_bwd(const float* ent, const float* rel, const float* norm_vect, float* grad_ent,
                                 float* grad_rel, float* grad_norm_vect, int dim, const int64_t* h,
                                 const int64_t* t, const int64_t* r, int64_t n, const float* grad_scores,
                                 void* stream);

/* TransD's scoring_function (models/translation.py:538-568): scores[i] = -||P(h~) + r~ - P(t~)||^2 with h~,
 * t~, r~ and the three projection vectors L2-normalised (eps 1e-12) and P(e~)[j] = (e~ . ep~) rp~[j] + e~[j] for
 * j < rel_dim.  Its own tables: ent / ent_proj [n_ent][ent_dim] (ent_emb.weight, ent_proj_vect.weight), rel /
 * rel_proj [n_rel][rel_dim] (rel_emb.weight, rel_proj_vect.weight).  rel_dim <= ent_dim <= 8192. */
int kge_transd_score_triples_fwd(const float* ent, const float* rel, const float* ent_proj, const float* rel_proj,
                                 int ent_dim, int rel_dim, const int64_t* h, const int64_t* t, const int64_t* r,
                                 int64_t n, float* scores, void* stream);
/* accumulates d(sum_i grad_scores[i] * scores[i]) / d(tables) into the four gradient tables */
int kge_transd_score_triples_bwd(const float* ent, const float* rel, const float* ent_proj, const float* rel_proj,
                                 float* grad_ent, float* grad_rel, float* grad_ent_proj, float* grad_rel_proj,
                                 int ent_dim, int rel_dim, const int64_t* h, const int64_t* t, const int64_t* r,
                                 int64_t n, const float* grad_scores, void* stream);

/* BernoulliNegativeSampler.corrupt_batch (sampling.py:278-327): nh/nt of length b*n_neg laid
 * out as n_neg blocks of the batch; negative j of fact i corrupts the head with probability
 * bern_probs[r[i]] else the tail, replacement uniform on [1, n_ent).  Counter-based RNG
 * (Philox4x32-10, key = seed, counter = (j*b+i, offset)). */
int kge_corrupt_batch(const int64_t* h, const int64_t* t, const int64_t* r, int64_t b,
                      int32_t n_neg, const float* bern_probs, int64_t n_ent, uint64_t seed,
                      uint64_t offset, int64_t* nh, int64_t* nt, void* stream);

/* MarginLoss (utils/losses.py:12-44): loss += sum_i max(0, margin - pos[i] + neg[i]). */
int kge_margin_loss_fwd(const float* pos, const float* neg, int64_t n, float margin, float* loss,
                        void* stream);
int kge_margin_loss_bwd(const float* pos, const float* neg, int64_t n, float margin,
                        const float* grad_loss, float* grad_pos, float* grad_neg, void* stream);

/* LogisticLoss (utils/losses.py:47-78: SoftMarginLoss(reduction='sum') on (pos, +1) and (neg, -1))
 * and BinaryCrossEntropyLoss (utils/losses.py:81-112: BCELoss(sum) of sigmoid(pos) vs 1 and
 * sigmoid(neg) vs 0, log clamped at -100 as torch does):
 *   kind 1: loss += sum_i log(1 + exp(-pos[i])) + log(1 + exp(neg[i]))
 *   kind 2: loss += sum_i -max(log(sig(pos[i])), -100) - max(log(1 - sig(neg[i])), -100)
 * Kind 0 (MarginLoss) is a loss kind of the fused step only (kge_margin_step_args_t.loss_kind). */
#define KGE_LOSS_MARGIN 0
#define KGE_LOSS_LOGISTIC 1
#define KGE_LOSS_BCE 2
int kge_pair_loss_fwd(int kind, const float* pos, const float* neg, int64_t n, float* loss, void* stream);
int kge_pair_loss_bwd(int kind, const float* pos, const float* neg, int64_t n, const float* grad_loss,
                      float* grad_pos, float* grad_neg, void* stream);

/* Fused training step = corrupt_batch + Model.forward (models/interfaces.py:39-82) +
 * the loss in one kernel: one warp per positive triple scores it and its n_neg negatives;
 * no (b*n_neg) index or score tensor is materialised unless the optional outputs are given.
 * Negatives: nh/nt if non-NULL (deterministic mode), else drawn in-kernel exactly as
 * kge_corrupt_batch would with the same (seed, offset).
 *
 * Loss (loss_kind): KGE_LOSS_MARGIN (MarginLoss(margin)), KGE_LOSS_LOGISTIC (LogisticLoss) or
 * KGE_LOSS_BCE (BinaryCrossEntropyLoss), summed over every (positive i, negative j) pair with the
 * per-pair terms of kge_pair_loss_fwd; margin is ignored unless loss_kind == KGE_LOSS_MARGIN.  Any
 * other kind returns KGE_ERR_ARG.  A zero-initialised loss_kind is the margin step of ABI 10.
 *
 * Entity-sharded step (hrows != NULL).  The entity table is range-partitioned: tb.ent0 / ent1 hold
 * the rows [ent_lo, ent_lo + n_rows) (n_rows = 0 is valid), n_ent is the GLOBAL entity count the draws
 * use, and hrows / trows are the positives' rows [b][planes][dim] as kge_gather_rows lays them out
 * (summed over the ranks).  Every rank makes the same draws; a negative is scored only by the rank
 * that holds its replaced entity, so summing `loss` over the ranks gives the unsharded loss.
 * Backward: the replaced rows' gradients go into g->ent0 / ent1 (local rows), the gradients of the
 * positives' h / t rows (also the intact entity of every negative) into grad_hrows / grad_trows
 * [b][planes][dim] (zeroed by the caller, added into), the relation gradients into g->rel0 / rel1.
 * Each of these is linear in the set of negatives: summing grad_hrows, grad_trows and the relation
 * gradients over the ranks, then adding the rows of grad_hrows / grad_trows into the entity gradient
 * (kge_scatter_rows_add) gives the unsharded gradient.  In this mode nh / nt, pos_out, neg_out,
 * nh_out, nt_out must be NULL, trows is required and, in backward, grad_hrows / grad_trows;
 * anything else returns KGE_ERR_ARG.  hrows == NULL: the unsharded step (ent_lo, n_rows, trows,
 * grad_hrows, grad_trows are ignored). */
typedef struct {
  kge_tables_t tb;
  int32_t n_neg;
  float margin;
  int64_t b;
  int64_t n_ent;
  const int64_t* h; const int64_t* t; const int64_t* r;
  const int64_t* nh; const int64_t* nt; /* optional external negatives */
  const float* bern_probs;              /* required when nh == NULL */
  uint64_t seed, offset;
  float* loss;                          /* 1 float, += */
  float* pos_out; float* neg_out;       /* optional */
  int64_t* nh_out; int64_t* nt_out;     /* optional */
  void* stream;
  int64_t ent_lo;                       /* sharded: global id of row 0 of tb.ent0 / ent1 */
  int64_t n_rows;                       /* sharded: rows held */
  const float* hrows; const float* trows;   /* sharded: [b][planes][dim] positive rows, or NULL */
  float* grad_hrows; float* grad_trows;     /* sharded backward: [b][planes][dim], += */
  int32_t loss_kind;                    /* KGE_LOSS_MARGIN (0), KGE_LOSS_LOGISTIC or KGE_LOSS_BCE */
} kge_margin_step_args_t;
int kge_margin_step_fwd(const kge_margin_step_args_t* a);
/* grad_loss: device pointer to the upstream gradient of the scalar loss */
int kge_margin_step_bwd(const kge_margin_step_args_t* a, const kge_grads_t* g,
                        const float* grad_loss);
/* The inverse of kge_gather_rows for gradients: grad_plane[idx[i] - ent_lo] += rows[i][plane] for
 * every i < n with ent_lo <= idx[i] < ent_lo + n_rows (atomics: ids may repeat); other ids are
 * ignored.  rows: [n][planes][dim]; grad1 for two- and three-plane models (plane 2 at
 * grad1 + (grad1 - grad0)). */
int kge_scatter_rows_add(int model, float* grad0, float* grad1, int64_t ent_lo, int64_t n_rows, int dim,
                         const int64_t* idx, int64_t n, const float* rows, void* stream);

/* ---- relation-corrupting negatives (BernoulliRelationNegativeSampler, sampling.py:507-553) ----------
 * kge_corrupt_batch_rel: nh / nt / nr of length b*n_neg in n_neg blocks of the batch.  Negative j of fact
 * i keeps its entities and replaces its relation, uniform on [1, n_rel), with probability 1 - rel_share;
 * otherwise it replaces the head with probability bern_probs[r[i]], else the tail, uniform on [1, n_ent),
 * and keeps its relation.  Exactly one position changes; true triples are not rejected.  Philox4x32-10
 * as kge_corrupt_batch (key = seed, counter = (j*b+i, offset)): words x, y decide and draw the entity as
 * there, word z decides entity (below rel_share) or relation, word w draws the relation -- so
 * rel_share = 1 gives kge_corrupt_batch's nh / nt.  0 <= rel_share <= 1; n_rel >= 2 unless rel_share = 1.
 *
 * kge_rel_step_fwd / _bwd: the fused step of kge_margin_step_fwd / _bwd with these negatives drawn in the
 * kernel at (seed, offset), exactly as kge_corrupt_batch_rel draws them, or taken from base.nh / base.nt
 * / nr (all three or none; any positions may change).  nr_out (optional, unsharded only) receives the
 * relations of the negatives next to base.nh_out / base.nt_out.  A negative scores (nh, nt, nr); its
 * gradient goes to those rows.  Entity-sharded (base.hrows != NULL): an entity negative is scored by the
 * rank holding its replaced entity as in kge_margin_step_fwd, a relation negative by the rank holding the
 * positive's HEAD, from hrows / trows, its entity gradients into grad_hrows / grad_trows and its relation
 * gradient into g->rel0 / rel1 -- the buffers the caller already sums over the ranks.  The argument rules
 * are those of kge_margin_step_fwd / _bwd, plus: n_rel >= 1, n_rel >= 2 unless rel_share >= 1,
 * rel_share in [0, 1], nr non-NULL exactly when base.nh is, and nr / nr_out NULL when sharded. */
int kge_corrupt_batch_rel(const int64_t* h, const int64_t* t, const int64_t* r, int64_t b, int32_t n_neg,
                          const float* bern_probs, int64_t n_ent, int64_t n_rel, float rel_share, uint64_t seed,
                          uint64_t offset, int64_t* nh, int64_t* nt, int64_t* nr, void* stream);
typedef struct {
  kge_margin_step_args_t base;
  int64_t n_rel;                        /* relations in the table: the relation draw is uniform on [1, n_rel) */
  float rel_share;                      /* probability that a negative replaces an entity */
  const int64_t* nr;                    /* external negatives' relations (with base.nh / base.nt), or NULL */
  int64_t* nr_out;                      /* optional: relations of the negatives (b*n_neg) */
} kge_rel_step_args_t;
int kge_rel_step_fwd(const kge_rel_step_args_t* a);
int kge_rel_step_bwd(const kge_rel_step_args_t* a, const kge_grads_t* g, const float* grad_loss);

/* ---- positional negatives (PositionalNegativeSampler, sampling.py:330-503) ------------------------------
 * kge_pos_step_fwd / _bwd: the fused step of kge_margin_step_fwd / _bwd with each negative drawn in the kernel
 * from the entities seen in its position for its relation.  The candidates are two CSR arrays per side:
 * relation r's heads are head_ents[head_offs[r] .. head_offs[r+1]), sorted, and likewise for tails.  Philox4x32-10
 * as kge_corrupt_batch (key = seed, counter = (j*b+i, offset)): word x replaces the head iff
 * (x >> 8) / 2^24 < bern_probs[r[i]], else the tail; word y picks the replacement ents[offs[r] + ((y n) >> 32)],
 * n = offs[r+1] - offs[r], or, when that slice is empty, (y n_ent) >> 32, uniform on [0, n_ent) -- entity 0
 * included, as in the reference.  Exactly one end is replaced; true triples are not rejected.  base.nh_out /
 * base.nt_out (optional, unsharded only) receive the negatives.  Entity-sharded (base.hrows != NULL): every
 * rank makes the same draws and a negative is scored by the rank holding its replaced entity, as in
 * kge_margin_step_fwd.  The argument rules are those of kge_margin_step_fwd / _bwd, plus: n_rel >= 1, both
 * offset arrays given (n_rel + 1 entries each), an ents array NULL only when all its slices are empty, and
 * base.nh / base.nt NULL (no caller negatives).  The caller guarantees r[i] < n_rel, non-decreasing offsets
 * and stored entities < base.n_ent. */
typedef struct {
  kge_margin_step_args_t base;
  int64_t n_rel;                        /* relations the CSR arrays cover */
  const int64_t* head_offs;             /* (n_rel + 1) offsets into head_ents */
  const int64_t* head_ents;             /* candidate heads, sorted within each relation */
  const int64_t* tail_offs;             /* (n_rel + 1) offsets into tail_ents */
  const int64_t* tail_ents;             /* candidate tails, sorted within each relation */
} kge_pos_step_args_t;
int kge_pos_step_fwd(const kge_pos_step_args_t* a);
int kge_pos_step_bwd(const kge_pos_step_args_t* a, const kge_grads_t* g, const float* grad_loss);

/* ---- data redundancy (torchkge/utils/data_redundancy.py: duplicates, count_triplets) ------------------
 * kge_cooccurrence: relation co-occurrence counts over two sets of facts.  Each side is a sorted array of
 * distinct keys (h * n_ent + t) * n_rel + r, cut into segments of equal (h, t): segment s holds keys
 * [offs[s], offs[s+1]) and pairs[s] = h * n_ent + t, ascending in s.  For every left segment (h, t) whose
 * partner -- the right segment of (h, t), or of (t, h) when flip != 0 -- exists, every key r_a of the left
 * segment and r_b of the partner add 1 to counts[r_a * n_rel + r_b] (n_rel x n_rel, uint64, zeroed by the
 * caller); upper != 0 keeps only r_a < r_b.  So counts[a][b] = |{(h, t) of a} & {(h, t) of b}|, or with
 * flip = |{(h, t) of a} & {(t, h) of b}|, self-loops included.  Arguments: n_ent >= 1, n_rel >= 1, every
 * pointer non-NULL; the caller guarantees the key layout above.  n_left == 0 or n_right == 0 is a no-op. */
int kge_cooccurrence(const int64_t* left_keys, const int64_t* left_offs, const int64_t* left_pairs, int64_t n_left,
                     const int64_t* right_keys, const int64_t* right_offs, const int64_t* right_pairs, int64_t n_right,
                     int64_t n_ent, int64_t n_rel, int flip, int upper, uint64_t* counts, void* stream);

/* ---- measurement hook ------------------------------------------------------------------
 * When enabled, the dominant kernels of kge_rank_side / kge_score_all are bracketed by CUDA
 * events recorded on the launch stream: kind 0 = scalar dense scan, 1 = tensor-core scan,
 * 2 = exact re-scoring of the near-tie list.  kge_scan_timing_read() synchronises the events
 * of one kind, returns the number of launches and their summed device time since the last
 * read, and clears that record.  Used by bench.py for the roofline figure; off by default
 * (no events are created). */
int kge_scan_timing_enable(int on);
int kge_scan_timing_read(int kind, int64_t* launches, double* total_ms);

#ifdef __cplusplus
}
#endif
#endif /* KGE_B200_H */
