// Internal launch interface of the training-side kernels (train.cu).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace kge {

struct TrainTables {
  const float* ent0;  // (n_ent, dim)
  const float* ent1;  // second entity plane (ComplEx / RotatE) or nullptr
  const float* rel0;  // (n_rel, dim) or RESCAL (n_rel, dim*dim)
  const float* rel1;  // second relation plane or nullptr
};

struct TrainGrads {
  float* ent0;
  float* ent1;
  float* rel0;
  float* rel1;
};

struct MarginStepParams {
  int model;
  int dim;
  int n_neg;
  float margin;
  long long b;      // positives
  long long n_ent;
  TrainTables tb;
  const int64_t* h;
  const int64_t* t;
  const int64_t* r;
  const int64_t* nh;  // external negatives (b * n_neg, blocks of b) or nullptr -> Philox
  const int64_t* nt;
  const float* probs;  // Bernoulli head-corruption probability per relation (Philox mode)
  uint64_t seed;
  uint64_t offset;
  float* loss;     // 1 float, +=
  float* pos_out;  // optional (b)
  float* neg_out;  // optional (b * n_neg)
  int64_t* nh_out;  // optional
  int64_t* nt_out;
  // Entity-sharded step (hrows != nullptr): tb.ent0 / ent1 hold rows [ent_lo, ent_lo + n_rows) of a
  // range-partitioned table, n_ent is the global count the draws use, the positive rows come from
  // hrows / trows and only the negatives whose replaced entity is held here are scored.
  long long ent_lo;
  long long n_rows;
  const float* hrows;  // [b][planes][dim]
  const float* trows;
  float* grad_hrows;   // [b][planes][dim], +=
  float* grad_trows;
  int loss_kind;       // KGE_LOSS_MARGIN / _LOGISTIC / _BCE; margin is used by the margin loss only
  // Relation-corrupting step (n_rel > 0, BernoulliRelationNegativeSampler): a negative replaces the
  // relation with probability 1 - rel_share (draw_rel), else the head or the tail.  External negatives
  // then come with nr; nr_out receives the relations of the negatives.  n_rel == 0: the entity step.
  long long n_rel;
  float rel_share;
  const int64_t* nr;
  int64_t* nr_out;
};

// Positional step (head_offs != nullptr, PositionalNegativeSampler): the replacement of a negative of
// relation r comes from the sorted slice [offs[r], offs[r + 1]) of ents on its side (draw_pos), or is uniform
// on [0, n_ent) when that slice is empty.  All nullptr: the entity or relation step.  A kernel parameter of its
// own, after the others, so that MarginStepParams -- and the code of the kernels that never draw positionally --
// stay as they are.
struct PosCSR {
  const int64_t* head_offs;
  const int64_t* head_ents;
  const int64_t* tail_offs;
  const int64_t* tail_ents;
};

cudaError_t launch_score_triples_fwd(int model, int dim, const TrainTables& tb, const int64_t* h,
                                     const int64_t* t, const int64_t* r, int64_t n, float* out,
                                     cudaStream_t st);
cudaError_t launch_score_triples_bwd(int model, int dim, const TrainTables& tb, const TrainGrads& gr,
                                     const int64_t* h, const int64_t* t, const int64_t* r, int64_t n,
                                     const float* gout, cudaStream_t st);
// TransH scoring_function (translation.py:183-202) on its own tables, forward and backward
cudaError_t launch_transh_score_fwd(const float* ent, const float* rel, const float* norm_vect, int dim,
                                    const int64_t* h, const int64_t* t, const int64_t* r, int64_t n, float* out,
                                    cudaStream_t st);
cudaError_t launch_transh_score_bwd(const float* ent, const float* rel, const float* norm_vect, float* g_ent,
                                    float* g_rel, float* g_norm_vect, int dim, const int64_t* h, const int64_t* t,
                                    const int64_t* r, int64_t n, const float* gout, cudaStream_t st);
// TransD scoring_function (translation.py:538-568) on its own tables, forward and backward
cudaError_t launch_transd_score_fwd(const float* ent, const float* rel, const float* ent_proj,
                                    const float* rel_proj, int ent_dim, int rel_dim, const int64_t* h,
                                    const int64_t* t, const int64_t* r, int64_t n, float* out, cudaStream_t st);
cudaError_t launch_transd_score_bwd(const float* ent, const float* rel, const float* ent_proj,
                                    const float* rel_proj, float* g_ent, float* g_rel, float* g_ent_proj,
                                    float* g_rel_proj, int ent_dim, int rel_dim, const int64_t* h, const int64_t* t,
                                    const int64_t* r, int64_t n, const float* gout, cudaStream_t st);
cudaError_t launch_corrupt_batch(const int64_t* h, const int64_t* t, const int64_t* r, int64_t b,
                                 int n_neg, const float* probs, int64_t n_ent, uint64_t seed,
                                 uint64_t offset, int64_t* nh, int64_t* nt, cudaStream_t st);
// BernoulliRelationNegativeSampler.corrupt_batch: draw_rel per negative, (nh, nt, nr) out
cudaError_t launch_corrupt_batch_rel(const int64_t* h, const int64_t* t, const int64_t* r, int64_t b,
                                     int n_neg, const float* probs, int64_t n_ent, int64_t n_rel, float rel_share,
                                     uint64_t seed, uint64_t offset, int64_t* nh, int64_t* nt, int64_t* nr,
                                     cudaStream_t st);
// pos: the positional step's candidates (PosCSR{} for the entity and relation steps)
cudaError_t launch_margin_step_fwd(const MarginStepParams& a, cudaStream_t st, const PosCSR& pos = PosCSR{});
cudaError_t launch_margin_step_bwd(const MarginStepParams& a, const TrainGrads& gr, const float* gloss,
                                   cudaStream_t st, const PosCSR& pos = PosCSR{});
cudaError_t launch_scatter_rows_add(float* grad0, float* grad1, int planes, int64_t ent_lo, int64_t n_rows,
                                    int dim, const int64_t* idx, int64_t n, const float* rows, cudaStream_t st);
// MarginLoss / LogisticLoss / BinaryCrossEntropyLoss on score arrays (kind: KGE_LOSS_*; margin is used by
// the margin loss only)
cudaError_t launch_pair_loss_fwd(int kind, float margin, const float* pos, const float* neg, int64_t n,
                                 float* loss, cudaStream_t st);
cudaError_t launch_pair_loss_bwd(int kind, float margin, const float* pos, const float* neg, int64_t n,
                                 const float* gloss, float* gpos, float* gneg, cudaStream_t st);

}  // namespace kge
