// Training-side kernels: per-triple scoring (Model.scoring_function), Bernoulli corruption
// (BernoulliNegativeSampler.corrupt_batch), the losses (MarginLoss, LogisticLoss,
// BinaryCrossEntropyLoss) and the fused sample + score + loss step, each with its backward.
//
// Reference bodies replaced: models/translation.py:69-81, models/bilinear.py:60-71, 188-199,
// 460-473, models/interfaces.py:39-82, sampling.py:278-327, utils/losses.py:12-44.
//
// These paths are gather-bound (a few 4d-byte rows per triple, random rows): one warp owns
// one triple (or one positive with all its negatives), lanes stride over the embedding
// index so every row read is a run of coalesced 128-B segments, and the per-triple
// reductions (L2 norms, dot products) are warp-shuffle trees.  Parity with the reference is
// by tolerance here (1e-5 relative on scores / loss, SURVEY.md section 8d), so fused
// multiply-adds and tree reductions are allowed, unlike in the ranking kernels.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include <stdlib.h>
#include <type_traits>

#include "../../include/kge_b200.h"
#include "ptx.cuh"
#include "train.h"

namespace kge {

namespace {

constexpr float NORM_EPS = 1e-12f;  // torch.nn.functional.normalize default eps
constexpr int WARPS_PER_BLOCK = 4;

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ bool model_normalises(int model) {
  return model == KGE_TRANSE_L1 || model == KGE_TRANSE_L2 || model == KGE_DISTMULT ||
         model == KGE_RESCAL;
}

// ---- Philox4x32-10 (Salmon et al. 2011), counter = (idx, offset), key = seed -------------
__device__ __forceinline__ uint4 philox4x32(uint64_t seed, uint64_t offset, uint64_t idx) {
  uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
  uint32_t c0 = (uint32_t)idx, c1 = (uint32_t)(idx >> 32);
  uint32_t c2 = (uint32_t)offset, c3 = (uint32_t)(offset >> 32);
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
    const uint32_t n0 = hi1 ^ c1 ^ k0, n1 = lo1, n2 = hi0 ^ c3 ^ k1, n3 = lo0;
    c0 = n0; c1 = n1; c2 = n2; c3 = n3;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  return make_uint4(c0, c1, c2, c3);
}

// The draw of one negative: Bernoulli(p_r) decides head vs tail (returned), the replacement *e is
// uniform on [1, n_ent) -- entity 0 is never drawn and true triples are not rejected, as in
// sampling.py:318-325.  Both depend on (seed, offset, idx, p, n_ent) only, so every rank of a sharded
// step makes the same draw and the same head / tail decision.
__device__ __forceinline__ bool draw_one(uint64_t seed, uint64_t offset, uint64_t idx, float p,
                                         long long n_ent, long long* e_out) {
  const uint4 rnd = philox4x32(seed, offset, idx);
  const float u = (rnd.x >> 8) * (1.0f / 16777216.0f);  // [0, 1)
  const long long span = n_ent - 1;
  long long e = 1;
  if (span > 0) e = 1 + (long long)(((unsigned long long)rnd.y * (unsigned long long)span) >> 32);
  *e_out = e;
  return u < p;
}

// One corrupted triple (nh, nt) of the positive (h, t).
__device__ __forceinline__ void corrupt_one(uint64_t seed, uint64_t offset, uint64_t idx, float p,
                                            long long n_ent, long long h, long long t,
                                            long long* nh, long long* nt) {
  long long e;
  const bool head = draw_one(seed, offset, idx, p, n_ent, &e);
  *nh = head ? e : h;
  *nt = head ? t : e;
}

// The draw of one relation-corrupting negative (BernoulliRelationNegativeSampler, sampling.py:507-553).
// Words x and y are those of draw_one: Bernoulli(p_r) decides head vs tail, the entity is uniform on
// [1, n_ent).  Word z decides entity (u < rel_share) vs relation; word w picks the relation, uniform on
// [1, n_rel).  Since u < 1 always, rel_share = 1 gives draw_one's draws.  Returns the kind.
constexpr int NEG_TAIL = 0, NEG_HEAD = 1, NEG_REL = 2;

__device__ __forceinline__ int draw_rel(uint64_t seed, uint64_t offset, uint64_t idx, float p, float rel_share,
                                        long long n_ent, long long n_rel, long long* e_out) {
  const uint4 rnd = philox4x32(seed, offset, idx);
  const float u_ent = (rnd.z >> 8) * (1.0f / 16777216.0f);
  if (!(u_ent < rel_share)) {
    const long long span = n_rel - 1;
    long long r = 1;
    if (span > 0) r = 1 + (long long)(((unsigned long long)rnd.w * (unsigned long long)span) >> 32);
    *e_out = r;
    return NEG_REL;
  }
  const float u = (rnd.x >> 8) * (1.0f / 16777216.0f);
  const long long span = n_ent - 1;
  long long e = 1;
  if (span > 0) e = 1 + (long long)(((unsigned long long)rnd.y * (unsigned long long)span) >> 32);
  *e_out = e;
  return u < p ? NEG_HEAD : NEG_TAIL;
}

// One corrupted triple (nh, nt, nr) of the positive (h, t, r).
__device__ __forceinline__ void corrupt_one_rel(uint64_t seed, uint64_t offset, uint64_t idx, float p,
                                                float rel_share, long long n_ent, long long n_rel, long long h,
                                                long long t, long long r, long long* nh, long long* nt,
                                                long long* nr) {
  long long e;
  const int kind = draw_rel(seed, offset, idx, p, rel_share, n_ent, n_rel, &e);
  *nh = kind == NEG_HEAD ? e : h;
  *nt = kind == NEG_TAIL ? e : t;
  *nr = kind == NEG_REL ? e : r;
}

// The positional draw (PositionalNegativeSampler, sampling.py:476-501).  Word x decides head vs tail exactly
// as in draw_one.  Word y picks the replacement uniformly in the sorted candidate slice of relation r on that
// side, ents[lo + ((y n) >> 32)] with n its length, or, when the slice is empty, uniformly on [0, n_ent):
// unlike draw_one, entity 0 is drawn, as in the reference.  True triples are not rejected.  The draw depends
// on (seed, offset, idx, r, the candidate slices) only, so every rank of a sharded step makes it too.
// PosSlices holds relation r's two slices: every negative of a positive shares r, so its bounds are loaded
// once per positive.
struct PosSlices {
  const int64_t* head_ents;   // first candidate of each side's slice
  const int64_t* tail_ents;
  long long n_head, n_tail;   // slice lengths
};

__device__ __forceinline__ PosSlices pos_slices(const PosCSR& pc, long long r) {
  PosSlices s;
  const long long h0 = pc.head_offs[r], t0 = pc.tail_offs[r];
  s.n_head = pc.head_offs[r + 1] - h0;
  s.n_tail = pc.tail_offs[r + 1] - t0;
  s.head_ents = pc.head_ents + h0;   // an ents array may be NULL only when its slices are all empty
  s.tail_ents = pc.tail_ents + t0;
  return s;
}

__device__ __forceinline__ bool draw_pos(uint64_t seed, uint64_t offset, uint64_t idx, float p, long long n_ent,
                                         const PosSlices& s, long long* e_out) {
  const uint4 rnd = philox4x32(seed, offset, idx);
  const float u = (rnd.x >> 8) * (1.0f / 16777216.0f);
  const bool head = u < p;
  const long long n = head ? s.n_head : s.n_tail;
  const int64_t* ents = head ? s.head_ents : s.tail_ents;
  const unsigned long long y = rnd.y;
  *e_out = n > 0 ? (long long)ents[(y * (unsigned long long)n) >> 32] : (long long)((y * (unsigned long long)n_ent) >> 32);
  return head;
}

// ------------------------------------------------------------------------------------------
// Per-lane view of one triple.  Lane l owns embedding indices l, l+32, ...; `cnt` of them.
// RowPtrs: the rows it is scored from.  GradRows: the destination rows of its gradient, plane by
// plane, in the same layout.
// ------------------------------------------------------------------------------------------
template <class T>
struct Rows {
  T* h0; T* h1;  // head planes
  T* t0; T* t1;  // tail planes
  T* r0; T* r1;  // relation planes (RESCAL: r0 = matrix)
  T* h2; T* t2; T* r2;  // third planes (Analogy) or nullptr
};
using RowPtrs = Rows<const float>;
using GradRows = Rows<float>;

__device__ __forceinline__ float inv_norm_of(const float* row, int dim, int lane) {
  float s = 0.f;
  for (int k = lane; k < dim; k += 32) { const float v = row[k]; s = fmaf(v, v, s); }
  s = warp_sum(s);
  return 1.0f / fmaxf(sqrtf(s), NORM_EPS);
}

// torch.frac: the fractional part keeps the sign of its argument
__device__ __forceinline__ float frac_of(float v) { return v - truncf(v); }

// score of one triple; all lanes return the same value
__device__ float triple_score(int model, int dim, const RowPtrs& p, int lane, float* inv_h_out,
                              float* inv_t_out) {
  float inv_h = 1.f, inv_t = 1.f;
  if (model_normalises(model)) {
    inv_h = inv_norm_of(p.h0, dim, lane);
    inv_t = inv_norm_of(p.t0, dim, lane);
  }
  if (inv_h_out) *inv_h_out = inv_h;
  if (inv_t_out) *inv_t_out = inv_t;
  float s = 0.f;
  switch (model) {
    case KGE_TRANSE_L1:
      for (int k = lane; k < dim; k += 32) s += fabsf(p.h0[k] * inv_h + p.r0[k] - p.t0[k] * inv_t);
      return -warp_sum(s);
    case KGE_TRANSE_L2:
      for (int k = lane; k < dim; k += 32) {
        const float x = p.h0[k] * inv_h + p.r0[k] - p.t0[k] * inv_t;
        s = fmaf(x, x, s);
      }
      return -warp_sum(s);
    case KGE_DISTMULT:
      for (int k = lane; k < dim; k += 32) s = fmaf(p.h0[k] * inv_h * p.r0[k], p.t0[k] * inv_t, s);
      return warp_sum(s);
    case KGE_RESCAL:
      // s = sum_j (sum_i h_i M_ij) t_j ; lanes stride over j so M rows are read coalesced
      for (int j = lane; j < dim; j += 32) {
        float q = 0.f;
        for (int i = 0; i < dim; ++i) q = fmaf(p.h0[i] * inv_h, p.r0[(size_t)i * dim + j], q);
        s = fmaf(q, p.t0[j] * inv_t, s);
      }
      return warp_sum(s);
    case KGE_COMPLEX:
      for (int k = lane; k < dim; k += 32) {
        const float rh = p.h0[k], ih = p.h1[k], rt = p.t0[k], it = p.t1[k], rr = p.r0[k], ir = p.r1[k];
        s += rh * (rr * rt + ir * it) + ih * (rr * it - ir * rt);
      }
      return warp_sum(s);
    case KGE_ROTATE:
      for (int k = lane; k < dim; k += 32) {
        const float rh = p.h0[k], ih = p.h1[k], rt = p.t0[k], it = p.t1[k], rr = p.r0[k], ir = p.r1[k];
        const float a = rh * rr - ih * ir - rt, b = rh * ir + ih * rr - it;
        s += sqrtf(a * a + b * b);
      }
      return -warp_sum(s);
    case KGE_TORUSE_L1:   // translation.py:706-720: -diss(frac(h) + frac(r), frac(t)), dissimilarities.py:28-43
    case KGE_TORUSE_L2:
      for (int k = lane; k < dim; k += 32) {
        const float x = (frac_of(p.h0[k]) + frac_of(p.r0[k])) - frac_of(p.t0[k]);
        if (model == KGE_TORUSE_L1) { const float ax = fabsf(x); s += 2.f * fminf(ax, 1.f - ax); }
        else { const float x2 = x * x; s += 4.f * fminf(x2, 1.f - x2); }
      }
      return -warp_sum(s);
    case KGE_ANALOGY:   // bilinear.py:634-650: DistMult on the scalar plane + ComplEx on (real, imaginary)
      for (int k = lane; k < dim; k += 32) {
        const float rh = p.h1[k], ih = p.h2[k], rt = p.t1[k], it = p.t2[k], rr = p.r1[k], ir = p.r2[k];
        s += p.h0[k] * p.r0[k] * p.t0[k] + (rh * (rr * rt + ir * it) + ih * (rr * it - ir * rt));
      }
      return warp_sum(s);
    default: return 0.f;
  }
}

// ---- row pointers, built plane by plane: from a dense table, or (entity-sharded rows) the replaced
// entity from the local table and the rest from [b][planes][dim] buffers.  Planes a model does not
// have are nullptr; triple_score / triple_backward dereference only the ones it has.
__device__ __forceinline__ int ent_planes(int model) {
  return model == KGE_ANALOGY ? 3 : (model == KGE_COMPLEX || model == KGE_ROTATE ? 2 : 1);
}

template <class T>
struct Planes { T* p0; T* p1; T* p2; };

// plane pointers of the row at element offset `off` of a table with planes p0, p1 (a third plane
// follows at the same spacing, include/kge_b200.h)
template <class T>
__device__ __forceinline__ Planes<T> table_planes(T* p0, T* p1, int np, size_t off) {
  Planes<T> o;
  o.p0 = p0 + off;
  o.p1 = np > 1 ? p1 + off : nullptr;
  o.p2 = np > 2 ? p1 + (p1 - p0) + off : nullptr;
  return o;
}

// row w of a [b][np][dim] buffer (hrows / trows / grad_hrows / grad_trows)
template <class T>
__device__ __forceinline__ Planes<T> buf_planes(T* buf, int np, int dim, long long w) {
  T* base = buf + (size_t)w * np * dim;
  return table_planes(base, base + dim, np, 0);
}

// relation row r of the (replicated) relation tables
template <class T>
__device__ __forceinline__ Planes<T> rel_planes(int model, int dim, T* r0, T* r1, long long r) {
  const size_t rstride = model == KGE_RESCAL ? (size_t)dim * dim : (size_t)dim;
  return table_planes(r0, r1, ent_planes(model), (size_t)r * rstride);
}

template <class T>
__device__ __forceinline__ Rows<T> rows_of(const Planes<T>& h, const Planes<T>& t, const Planes<T>& r) {
  Rows<T> p;
  p.h0 = h.p0; p.h1 = h.p1; p.h2 = h.p2;
  p.t0 = t.p0; p.t1 = t.p1; p.t2 = t.p2;
  p.r0 = r.p0; p.r1 = r.p1; p.r2 = r.p2;
  return p;
}

// The rows of triple (h, t, r) in dense tables: RowPtrs from TrainTables, GradRows from TrainGrads.
template <class Tables>
__device__ __forceinline__ auto table_rows(int model, int dim, const Tables& tb, long long h, long long t,
                                           long long r) {
  const int np = ent_planes(model);
  return rows_of(table_planes(tb.ent0, tb.ent1, np, (size_t)h * dim),
                 table_planes(tb.ent0, tb.ent1, np, (size_t)t * dim),
                 rel_planes(model, dim, tb.rel0, tb.rel1, r));
}

// Gradient of one triple's score, scaled by g, added into the rows `d` (atomics: rows repeat).
// Through F.normalize:  d/dh = (G - h~ (h~ . G)) / max(|h|, eps)  with G = dscore/dh~.
__device__ void triple_backward(int model, int dim, const RowPtrs& p, const GradRows& d, float g, int lane) {
  if (g == 0.f) return;
  float* gh0 = d.h0;
  float* gt0 = d.t0;
  float* gr0 = d.r0;
  if (model == KGE_COMPLEX || model == KGE_ROTATE) {
    float* gh1 = d.h1;
    float* gt1 = d.t1;
    float* gr1 = d.r1;
    for (int k = lane; k < dim; k += 32) {
      const float rh = p.h0[k], ih = p.h1[k], rt = p.t0[k], it = p.t1[k], rr = p.r0[k], ir = p.r1[k];
      float d_rh, d_ih, d_rt, d_it, d_rr, d_ir;
      if (model == KGE_COMPLEX) {
        d_rh = rr * rt + ir * it; d_ih = rr * it - ir * rt;
        d_rt = rh * rr - ih * ir; d_it = rh * ir + ih * rr;
        d_rr = rh * rt + ih * it; d_ir = rh * it - ih * rt;
      } else {
        const float a = rh * rr - ih * ir - rt, b = rh * ir + ih * rr - it;
        const float m = sqrtf(a * a + b * b);
        const float da = m > 0.f ? -a / m : 0.f, db = m > 0.f ? -b / m : 0.f;
        d_rh = da * rr + db * ir; d_ih = -da * ir + db * rr;
        d_rt = -da; d_it = -db;
        d_rr = da * rh + db * ih; d_ir = -da * ih + db * rh;
      }
      atomicAdd(gh0 + k, g * d_rh); atomicAdd(gh1 + k, g * d_ih);
      atomicAdd(gt0 + k, g * d_rt); atomicAdd(gt1 + k, g * d_it);
      atomicAdd(gr0 + k, g * d_rr); atomicAdd(gr1 + k, g * d_ir);
    }
    return;
  }
  if (model == KGE_ANALOGY) {
    float* gh1 = d.h1;
    float* gt1 = d.t1;
    float* gr1 = d.r1;
    float* gh2 = d.h2;
    float* gt2 = d.t2;
    float* gr2 = d.r2;
    for (int k = lane; k < dim; k += 32) {
      const float sh = p.h0[k], st = p.t0[k], sr = p.r0[k];
      atomicAdd(gh0 + k, g * (sr * st)); atomicAdd(gt0 + k, g * (sh * sr)); atomicAdd(gr0 + k, g * (sh * st));
      const float rh = p.h1[k], ih = p.h2[k], rt = p.t1[k], it = p.t2[k], rr = p.r1[k], ir = p.r2[k];
      atomicAdd(gh1 + k, g * (rr * rt + ir * it)); atomicAdd(gh2 + k, g * (rr * it - ir * rt));
      atomicAdd(gt1 + k, g * (rh * rr - ih * ir)); atomicAdd(gt2 + k, g * (rh * ir + ih * rr));
      atomicAdd(gr1 + k, g * (rh * rt + ih * it)); atomicAdd(gr2 + k, g * (rh * it - ih * rt));
    }
    return;
  }
  if (model == KGE_TORUSE_L1 || model == KGE_TORUSE_L2) {
    // x = frac(h) + frac(r) - frac(t) (frac has unit slope); min(u, v) sends the gradient to the
    // smaller argument and, as torch.min does, half to each at an exact tie
    for (int k = lane; k < dim; k += 32) {
      const float x = (frac_of(p.h0[k]) + frac_of(p.r0[k])) - frac_of(p.t0[k]);
      float d;   // d score / d x
      if (model == KGE_TORUSE_L1) {
        const float ax = fabsf(x), sg = x > 0.f ? 1.f : (x < 0.f ? -1.f : 0.f);
        d = ax < 1.f - ax ? -2.f * sg : (ax > 1.f - ax ? 2.f * sg : 0.f);
      } else {
        const float x2 = x * x;
        d = x2 < 1.f - x2 ? -8.f * x : (x2 > 1.f - x2 ? 8.f * x : 0.f);
      }
      atomicAdd(gh0 + k, g * d); atomicAdd(gr0 + k, g * d); atomicAdd(gt0 + k, -g * d);
    }
    return;
  }
  // normalising models
  const float inv_h = inv_norm_of(p.h0, dim, lane), inv_t = inv_norm_of(p.t0, dim, lane);
  // pass 1: G . h~ and G . t~
  float dot_h = 0.f, dot_t = 0.f;
  for (int k = lane; k < dim; k += 32) {
    const float hn = p.h0[k] * inv_h, tn = p.t0[k] * inv_t;
    float Gh, Gt;
    if (model == KGE_DISTMULT) {
      Gh = p.r0[k] * tn; Gt = hn * p.r0[k];
    } else if (model == KGE_RESCAL) {
      float a = 0.f, b = 0.f;  // Gh_k = sum_j M_kj t_j ; Gt_k = sum_i h_i M_ik
      for (int j = 0; j < dim; ++j) {
        a = fmaf(p.r0[(size_t)k * dim + j], p.t0[j] * inv_t, a);
        b = fmaf(p.h0[j] * inv_h, p.r0[(size_t)j * dim + k], b);
      }
      Gh = a; Gt = b;
    } else {
      const float x = hn + p.r0[k] - tn;
      const float dx = model == KGE_TRANSE_L2 ? -2.f * x : (x > 0.f ? -1.f : (x < 0.f ? 1.f : 0.f));
      Gh = dx; Gt = -dx;
    }
    dot_h = fmaf(Gh, hn, dot_h); dot_t = fmaf(Gt, tn, dot_t);
  }
  dot_h = warp_sum(dot_h); dot_t = warp_sum(dot_t);
  // pass 2: scatter
  for (int k = lane; k < dim; k += 32) {
    const float hn = p.h0[k] * inv_h, tn = p.t0[k] * inv_t;
    float Gh, Gt;
    if (model == KGE_DISTMULT) {
      Gh = p.r0[k] * tn; Gt = hn * p.r0[k];
      atomicAdd(gr0 + k, g * hn * tn);
    } else if (model == KGE_RESCAL) {
      float a = 0.f, b = 0.f;
      for (int j = 0; j < dim; ++j) {
        a = fmaf(p.r0[(size_t)k * dim + j], p.t0[j] * inv_t, a);
        b = fmaf(p.h0[j] * inv_h, p.r0[(size_t)j * dim + k], b);
        atomicAdd(gr0 + (size_t)k * dim + j, g * hn * (p.t0[j] * inv_t));  // dM_kj = h_k t_j
      }
      Gh = a; Gt = b;
    } else {
      const float x = hn + p.r0[k] - tn;
      const float dx = model == KGE_TRANSE_L2 ? -2.f * x : (x > 0.f ? -1.f : (x < 0.f ? 1.f : 0.f));
      Gh = dx; Gt = -dx;
      atomicAdd(gr0 + k, g * dx);
    }
    atomicAdd(gh0 + k, g * (Gh - hn * dot_h) * inv_h);
    atomicAdd(gt0 + k, g * (Gt - tn * dot_t) * inv_t);
  }
}

// ---- TransH scoring_function (translation.py:183-202): with h~, t~, w~ the L2-normalised head, tail and
// normal vector of the relation, a = h~ . w~, b = t~ . w~,
//   x = (h~ - a w~) + r - (t~ - b w~),   score = -|x|^2.
// Its own tables (ent, rel, norm_vect) rather than a model code: the tables of the other models cannot carry it.
struct TransHRows {
  const float* h; const float* t; const float* r; const float* w;
  float ih, it, iw;   // 1 / max(|row|, eps)
  float a, b;         // h~ . w~ and t~ . w~
};

__device__ __forceinline__ TransHRows transh_rows(const float* ent, const float* rel, const float* nv, int dim,
                                                  long long h, long long t, long long r, int lane) {
  TransHRows p;
  p.h = ent + (size_t)h * dim; p.t = ent + (size_t)t * dim;
  p.r = rel + (size_t)r * dim; p.w = nv + (size_t)r * dim;
  p.ih = inv_norm_of(p.h, dim, lane); p.it = inv_norm_of(p.t, dim, lane); p.iw = inv_norm_of(p.w, dim, lane);
  float a = 0.f, b = 0.f;
  for (int k = lane; k < dim; k += 32) {
    const float wn = p.w[k] * p.iw;
    a = fmaf(p.h[k] * p.ih, wn, a);
    b = fmaf(p.t[k] * p.it, wn, b);
  }
  p.a = warp_sum(a); p.b = warp_sum(b);
  return p;
}

__device__ __forceinline__ float transh_x(const TransHRows& p, int k) {
  const float wn = p.w[k] * p.iw;
  return (p.h[k] * p.ih - p.a * wn) + p.r[k] - (p.t[k] * p.it - p.b * wn);
}

__global__ void transh_score_fwd_kernel(const float* __restrict__ ent, const float* __restrict__ rel,
                                        const float* __restrict__ nv, int dim, const int64_t* __restrict__ h,
                                        const int64_t* __restrict__ t, const int64_t* __restrict__ r, long long n,
                                        float* __restrict__ out) {
  const long long w = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= n) return;
  const TransHRows p = transh_rows(ent, rel, nv, dim, h[w], t[w], r[w], lane);
  float s = 0.f;
  for (int k = lane; k < dim; k += 32) { const float x = transh_x(p, k); s = fmaf(x, x, s); }
  s = warp_sum(s);
  if (lane == 0) out[w] = -s;
}

// With G = dscore/dx = -2x and c = w~ . G:
//   dscore/dh~ = G - c w~,   dscore/dt~ = -(G - c w~),   dscore/dr = G,   dscore/dw~ = -(a - b) G - c (h~ - t~),
// each then through F.normalize:  d/dv = (G_v - v~ (v~ . G_v)) / max(|v|, eps), where
//   h~ . G_h = h~.G - c a,   t~ . G_t = -(t~.G - c b),   w~ . G_w = -2 c (a - b).
__global__ void transh_score_bwd_kernel(const float* __restrict__ ent, const float* __restrict__ rel,
                                        const float* __restrict__ nv, float* __restrict__ g_ent,
                                        float* __restrict__ g_rel, float* __restrict__ g_nv, int dim,
                                        const int64_t* __restrict__ h, const int64_t* __restrict__ t,
                                        const int64_t* __restrict__ r, long long n, const float* __restrict__ gout) {
  const long long w = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= n) return;
  const float g = gout[w];
  if (g == 0.f) return;
  const long long hi = h[w], ti = t[w], ri = r[w];
  const TransHRows p = transh_rows(ent, rel, nv, dim, hi, ti, ri, lane);
  float c = 0.f, hg = 0.f, tg = 0.f;
  for (int k = lane; k < dim; k += 32) {
    const float G = -2.f * transh_x(p, k);
    c = fmaf(p.w[k] * p.iw, G, c);
    hg = fmaf(p.h[k] * p.ih, G, hg);
    tg = fmaf(p.t[k] * p.it, G, tg);
  }
  c = warp_sum(c); hg = warp_sum(hg); tg = warp_sum(tg);
  const float dot_h = hg - c * p.a, dot_t = -(tg - c * p.b), dot_w = -2.f * c * (p.a - p.b);
  float* gh = g_ent + (size_t)hi * dim;
  float* gt = g_ent + (size_t)ti * dim;
  float* gr = g_rel + (size_t)ri * dim;
  float* gw = g_nv + (size_t)ri * dim;
  for (int k = lane; k < dim; k += 32) {
    const float hn = p.h[k] * p.ih, tn = p.t[k] * p.it, wn = p.w[k] * p.iw;
    const float G = -2.f * transh_x(p, k);
    const float Gh = G - c * wn;
    const float Gw = -(p.a - p.b) * G - c * (hn - tn);
    atomicAdd(gh + k, g * (Gh - hn * dot_h) * p.ih);
    atomicAdd(gt + k, g * (-Gh - tn * dot_t) * p.it);
    atomicAdd(gr + k, g * G);
    atomicAdd(gw + k, g * (Gw - wn * dot_w) * p.iw);
  }
}

// ---- TransD scoring_function (translation.py:538-568): with h~, t~, r~, hp~, tp~, rp~ the L2-normalised
// head, tail, relation and their projection vectors, a = h~ . hp~, b = t~ . tp~ (over ent_dim),
//   x[j] = (a rp~[j] + h~[j]) + r~[j] - (b rp~[j] + t~[j])  for j < rel_dim,   score = -|x|^2.
// Its own tables (ent, rel, ent_proj, rel_proj) and two widths rather than a model code.
struct TransDRows {
  const float* h; const float* t; const float* hp; const float* tp;   // [ent_dim]
  const float* r; const float* rp;                                     // [rel_dim]
  float ih, it, ihp, itp, ir, irp;   // 1 / max(|row|, eps)
  float a, b;                        // h~ . hp~ and t~ . tp~
};

__device__ __forceinline__ TransDRows transd_rows(const float* ent, const float* rel, const float* ep,
                                                  const float* rpv, int ent_dim, int rel_dim, long long h,
                                                  long long t, long long r, int lane) {
  TransDRows p;
  p.h = ent + (size_t)h * ent_dim; p.t = ent + (size_t)t * ent_dim;
  p.hp = ep + (size_t)h * ent_dim; p.tp = ep + (size_t)t * ent_dim;
  p.r = rel + (size_t)r * rel_dim; p.rp = rpv + (size_t)r * rel_dim;
  p.ih = inv_norm_of(p.h, ent_dim, lane); p.it = inv_norm_of(p.t, ent_dim, lane);
  p.ihp = inv_norm_of(p.hp, ent_dim, lane); p.itp = inv_norm_of(p.tp, ent_dim, lane);
  p.ir = inv_norm_of(p.r, rel_dim, lane); p.irp = inv_norm_of(p.rp, rel_dim, lane);
  float a = 0.f, b = 0.f;
  for (int k = lane; k < ent_dim; k += 32) {
    a = fmaf(p.h[k] * p.ih, p.hp[k] * p.ihp, a);
    b = fmaf(p.t[k] * p.it, p.tp[k] * p.itp, b);
  }
  p.a = warp_sum(a); p.b = warp_sum(b);
  return p;
}

__device__ __forceinline__ float transd_x(const TransDRows& p, int j) {
  const float rpn = p.rp[j] * p.irp;
  return (p.a * rpn + p.h[j] * p.ih) + p.r[j] * p.ir - (p.b * rpn + p.t[j] * p.it);
}

__global__ void transd_score_fwd_kernel(const float* __restrict__ ent, const float* __restrict__ rel,
                                        const float* __restrict__ ep, const float* __restrict__ rpv, int ent_dim,
                                        int rel_dim, const int64_t* __restrict__ h, const int64_t* __restrict__ t,
                                        const int64_t* __restrict__ r, long long n, float* __restrict__ out) {
  const long long w = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= n) return;
  const TransDRows p = transd_rows(ent, rel, ep, rpv, ent_dim, rel_dim, h[w], t[w], r[w], lane);
  float s = 0.f;
  for (int j = lane; j < rel_dim; j += 32) { const float x = transd_x(p, j); s = fmaf(x, x, s); }
  s = warp_sum(s);
  if (lane == 0) out[w] = -s;
}

// With G = dscore/dx = -2x (rel_dim) and c = rp~ . G:
//   dscore/dh~ = [G, 0..] + c hp~,   dscore/dhp~ = c h~,   dscore/dt~ = -[G, 0..] - c tp~,   dscore/dtp~ = -c t~,
//   dscore/dr~ = G,   dscore/drp~ = (a - b) G,
// each then through F.normalize:  d/dv = (G_v - v~ (v~ . G_v)) / max(|v|, eps), where
//   h~ . G_h = h~[:rel_dim].G + c a,  hp~ . G_hp = c a,  t~ . G_t = -(t~[:rel_dim].G + c b),  tp~ . G_tp = -c b,
//   rp~ . G_rp = (a - b) c.
__global__ void transd_score_bwd_kernel(const float* __restrict__ ent, const float* __restrict__ rel,
                                        const float* __restrict__ ep, const float* __restrict__ rpv,
                                        float* __restrict__ g_ent, float* __restrict__ g_rel,
                                        float* __restrict__ g_ep, float* __restrict__ g_rpv, int ent_dim,
                                        int rel_dim, const int64_t* __restrict__ h, const int64_t* __restrict__ t,
                                        const int64_t* __restrict__ r, long long n, const float* __restrict__ gout) {
  const long long w = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= n) return;
  const float g = gout[w];
  if (g == 0.f) return;
  const long long hi = h[w], ti = t[w], ri = r[w];
  const TransDRows p = transd_rows(ent, rel, ep, rpv, ent_dim, rel_dim, hi, ti, ri, lane);
  float c = 0.f, hg = 0.f, tg = 0.f, rg = 0.f;
  for (int j = lane; j < rel_dim; j += 32) {
    const float G = -2.f * transd_x(p, j);
    c = fmaf(p.rp[j] * p.irp, G, c);
    hg = fmaf(p.h[j] * p.ih, G, hg);
    tg = fmaf(p.t[j] * p.it, G, tg);
    rg = fmaf(p.r[j] * p.ir, G, rg);
  }
  c = warp_sum(c); hg = warp_sum(hg); tg = warp_sum(tg); rg = warp_sum(rg);
  const float dot_h = hg + c * p.a, dot_hp = c * p.a, dot_t = -(tg + c * p.b), dot_tp = -c * p.b;
  const float dot_rp = (p.a - p.b) * c;
  float* gh = g_ent + (size_t)hi * ent_dim;
  float* gt = g_ent + (size_t)ti * ent_dim;
  float* ghp = g_ep + (size_t)hi * ent_dim;
  float* gtp = g_ep + (size_t)ti * ent_dim;
  for (int k = lane; k < ent_dim; k += 32) {
    const float hn = p.h[k] * p.ih, tn = p.t[k] * p.it, hpn = p.hp[k] * p.ihp, tpn = p.tp[k] * p.itp;
    const float G = k < rel_dim ? -2.f * transd_x(p, k) : 0.f;
    atomicAdd(gh + k, g * (G + c * hpn - hn * dot_h) * p.ih);
    atomicAdd(gt + k, g * (-G - c * tpn - tn * dot_t) * p.it);
    atomicAdd(ghp + k, g * (c * hn - hpn * dot_hp) * p.ihp);
    atomicAdd(gtp + k, g * (-c * tn - tpn * dot_tp) * p.itp);
  }
  float* gr = g_rel + (size_t)ri * rel_dim;
  float* grp = g_rpv + (size_t)ri * rel_dim;
  for (int j = lane; j < rel_dim; j += 32) {
    const float rn = p.r[j] * p.ir, rpn = p.rp[j] * p.irp;
    const float G = -2.f * transd_x(p, j);
    atomicAdd(gr + j, g * (G - rn * rg) * p.ir);
    atomicAdd(grp + j, g * ((p.a - p.b) * G - rpn * dot_rp) * p.irp);
  }
}

// ------------------------------------------------------------------------------------------
__global__ void score_triples_fwd_kernel(int model, int dim, TrainTables tb,
                                         const int64_t* __restrict__ h,
                                         const int64_t* __restrict__ t,
                                         const int64_t* __restrict__ r, long long n,
                                         float* __restrict__ out) {
  const long long w = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= n) return;
  const RowPtrs p = table_rows(model, dim, tb, h[w], t[w], r[w]);
  const float s = triple_score(model, dim, p, lane, nullptr, nullptr);
  if (lane == 0) out[w] = s;
}

__global__ void score_triples_bwd_kernel(int model, int dim, TrainTables tb, TrainGrads gr,
                                         const int64_t* __restrict__ h,
                                         const int64_t* __restrict__ t,
                                         const int64_t* __restrict__ r, long long n,
                                         const float* __restrict__ gout) {
  const long long w = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= n) return;
  const long long hi = h[w], ti = t[w], ri = r[w];
  const RowPtrs p = table_rows(model, dim, tb, hi, ti, ri);
  triple_backward(model, dim, p, table_rows(model, dim, gr, hi, ti, ri), gout[w], lane);
}

__global__ void corrupt_batch_kernel(const int64_t* __restrict__ h, const int64_t* __restrict__ t,
                                     const int64_t* __restrict__ r, long long b, int n_neg,
                                     const float* __restrict__ probs, long long n_ent,
                                     uint64_t seed, uint64_t offset, int64_t* __restrict__ nh,
                                     int64_t* __restrict__ nt) {
  const long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (gid >= b * n_neg) return;
  const long long i = gid % b;  // layout: n_neg blocks of the batch (sampling.py:313-314)
  long long a, c;
  corrupt_one(seed, offset, (uint64_t)gid, probs[r[i]], n_ent, h[i], t[i], &a, &c);
  nh[gid] = a; nt[gid] = c;
}

__global__ void corrupt_batch_rel_kernel(const int64_t* __restrict__ h, const int64_t* __restrict__ t,
                                         const int64_t* __restrict__ r, long long b, int n_neg,
                                         const float* __restrict__ probs, long long n_ent, long long n_rel,
                                         float rel_share, uint64_t seed, uint64_t offset, int64_t* __restrict__ nh,
                                         int64_t* __restrict__ nt, int64_t* __restrict__ nr) {
  const long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (gid >= b * n_neg) return;
  const long long i = gid % b;
  long long a, c, q;
  corrupt_one_rel(seed, offset, (uint64_t)gid, probs[r[i]], rel_share, n_ent, n_rel, h[i], t[i], r[i], &a, &c, &q);
  nh[gid] = a; nt[gid] = c; nr[gid] = q;
}

// Negative idx of the positive (hi, ti, ri) in the generic kernels: the caller's (nh, nt[, nr]), else a
// Philox draw -- draw_rel in a relation-corrupting step (a.n_rel > 0), draw_one otherwise.
__device__ __forceinline__ void step_negative(const MarginStepParams& a, long long idx, float p_head, long long hi,
                                              long long ti, long long ri, long long* nh, long long* nt,
                                              long long* nr) {
  if (a.nh) {
    *nh = a.nh[idx]; *nt = a.nt[idx]; *nr = a.nr ? a.nr[idx] : ri;
  } else if (a.n_rel > 0) {
    corrupt_one_rel(a.seed, a.offset, (uint64_t)idx, p_head, a.rel_share, a.n_ent, a.n_rel, hi, ti, ri, nh, nt, nr);
  } else {
    corrupt_one(a.seed, a.offset, (uint64_t)idx, p_head, a.n_ent, hi, ti, nh, nt);
    *nr = ri;
  }
}

// The generic kernels' negative: the positional draw in a positional step (pc.head_offs set; ps: the
// positive's slices), else step_negative.
__device__ __forceinline__ void generic_negative(const MarginStepParams& a, const PosCSR& pc, const PosSlices& ps,
                                                 long long idx, float p_head, long long hi, long long ti, long long ri,
                                                 long long* nh, long long* nt, long long* nr) {
  if (pc.head_offs) {
    long long e;
    const bool head = draw_pos(a.seed, a.offset, (uint64_t)idx, p_head, a.n_ent, ps, &e);
    *nh = head ? e : hi; *nt = head ? ti : e; *nr = ri;
  } else {
    step_negative(a, idx, p_head, hi, ti, ri, nh, nt, nr);
  }
}

__device__ __forceinline__ PosSlices generic_slices(const PosCSR& pc, long long r) {
  return pc.head_offs ? pos_slices(pc, r) : PosSlices{nullptr, nullptr, 0, 0};
}

// ---- per-pair loss terms: the one statement of each loss, used by pair_loss_fwd / _bwd_kernel and
// by every fused step (kind: KGE_LOSS_*, a runtime value or a template constant).
//   margin  : max(0, margin - pos + neg)                    (MarginRankingLoss, target +1, sum)
//   logistic: softplus(-pos) + softplus(neg), softplus(x) = max(x, 0) + log1p(exp(-|x|))
//             (SoftMarginLoss(sum) on (pos, +1) and (neg, -1), utils/losses.py:47-78)
//   bce     : -max(log(sig(pos)), -100) - max(log(1 - sig(neg)), -100), sig in fp32 as torch does
//             (BCELoss(sum) of sig(pos) vs 1 and sig(neg) vs 0, utils/losses.py:81-112)
__device__ __forceinline__ float softplus_f(float x) { return fmaxf(x, 0.f) + log1pf(expf(-fabsf(x))); }
__device__ __forceinline__ float sigmoid_f(float x) { return 1.0f / (1.0f + expf(-x)); }

__device__ __forceinline__ float pair_loss_term(int kind, float margin, float pos, float neg) {
  if (kind == KGE_LOSS_MARGIN) return fmaxf(0.f, margin - pos + neg);
  if (kind == KGE_LOSS_LOGISTIC) return softplus_f(-pos) + softplus_f(neg);
  const float pp = sigmoid_f(pos), pn = sigmoid_f(neg);
  return -fmaxf(logf(pp), -100.f) - fmaxf(logf(1.0f - pn), -100.f);
}

// g * d(term)/d pos and g * d(term)/d neg of one pair, as torch's backward computes them
__device__ __forceinline__ void pair_loss_grads(int kind, float margin, float g, float pos, float neg,
                                                float* gpos, float* gneg) {
  if (kind == KGE_LOSS_MARGIN) {   // same sub-gradient as torch: zero at the kink
    const bool on = margin - pos + neg > 0.f;
    *gpos = on ? -g : 0.f;
    *gneg = on ? g : 0.f;
    return;
  }
  const float pp = sigmoid_f(pos), pn = sigmoid_f(neg);
  if (kind == KGE_LOSS_LOGISTIC) {
    *gpos = g * (pp - 1.0f);   // d/dx log(1 + exp(-x)) = -sig(-x) = sig(x) - 1
    *gneg = g * pn;            // d/dx log(1 + exp(x))  = sig(x)
  } else {
    // torch's BCELoss backward: (p - y) / max(p (1 - p), 1e-12), chained with dp/dx = p (1 - p); a
    // saturated sigmoid (p = 0 or 1 exactly) gives exactly 0
    *gpos = g * (pp - 1.0f) / fmaxf(pp * (1.0f - pp), 1e-12f) * (pp * (1.0f - pp));
    *gneg = g * pn / fmaxf(pn * (1.0f - pn), 1e-12f) * (pn * (1.0f - pn));
  }
}

// Fused step, forward: one warp per positive triple.
//   loss += sum_j pair_loss_term(pos_i, neg_ij)
// Negatives come from (nh, nt) if given, else from Philox; optionally written out.
__global__ void margin_step_fwd_kernel(MarginStepParams a, PosCSR pc) {
  const long long w = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= a.b) return;
  const long long hi = a.h[w], ti = a.t[w], ri = a.r[w];
  const RowPtrs pp = table_rows(a.model, a.dim, a.tb, hi, ti, ri);
  const float pos = triple_score(a.model, a.dim, pp, lane, nullptr, nullptr);
  if (lane == 0 && a.pos_out) a.pos_out[w] = pos;
  const float p_head = a.nh ? 0.f : a.probs[ri];
  const PosSlices ps = generic_slices(pc, ri);
  float loss = 0.f;
  for (int j = 0; j < a.n_neg; ++j) {
    const long long idx = (long long)j * a.b + w;
    long long nh, nt, nr;
    generic_negative(a, pc, ps, idx, p_head, hi, ti, ri, &nh, &nt, &nr);
    const RowPtrs pn = table_rows(a.model, a.dim, a.tb, nh, nt, nr);
    const float neg = triple_score(a.model, a.dim, pn, lane, nullptr, nullptr);
    if (lane == 0) {
      if (a.neg_out) a.neg_out[idx] = neg;
      if (a.nh_out) { a.nh_out[idx] = nh; a.nt_out[idx] = nt; }
      if (a.nr_out) a.nr_out[idx] = nr;
      loss += pair_loss_term(a.loss_kind, a.margin, pos, neg);
    }
  }
  if (lane == 0) atomicAdd(a.loss, loss);
}

// Fused step, backward: recompute the same negatives and scores; pair j sends g dl/dneg to the
// negative triple, and the positive triple gets the sum over j of g dl/dpos in one call (the margin
// loss: +g per active hinge to the negative, -g times the active count to the positive).
__global__ void margin_step_bwd_kernel(MarginStepParams a, TrainGrads gr, const float* gloss, PosCSR pc) {
  const long long w = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= a.b) return;
  const float g = *gloss;
  const long long hi = a.h[w], ti = a.t[w], ri = a.r[w];
  const RowPtrs pp = table_rows(a.model, a.dim, a.tb, hi, ti, ri);
  const float pos = triple_score(a.model, a.dim, pp, lane, nullptr, nullptr);
  const float p_head = a.nh ? 0.f : a.probs[ri];
  const PosSlices ps = generic_slices(pc, ri);
  double gpos_sum = 0.0;   // thousands of non-integer dl/dpos terms (logistic, BCE): fp32 would drift
  for (int j = 0; j < a.n_neg; ++j) {
    const long long idx = (long long)j * a.b + w;
    long long nh, nt, nr;
    generic_negative(a, pc, ps, idx, p_head, hi, ti, ri, &nh, &nt, &nr);
    const RowPtrs pn = table_rows(a.model, a.dim, a.tb, nh, nt, nr);
    const float neg = triple_score(a.model, a.dim, pn, lane, nullptr, nullptr);
    float gp, gn;
    pair_loss_grads(a.loss_kind, a.margin, 1.f, pos, neg, &gp, &gn);
    gpos_sum += gp;
    triple_backward(a.model, a.dim, pn, table_rows(a.model, a.dim, gr, nh, nt, nr), g * gn, lane);
  }
  triple_backward(a.model, a.dim, pp, table_rows(a.model, a.dim, gr, hi, ti, ri), g * (float)gpos_sum, lane);
}

// Entity-sharded fused step (a.hrows set), one warp per positive.  Every rank runs the same draws;
// a negative is scored here only if its replaced entity e lies in [ent_lo, ent_lo + n_rows).  Its
// rows: e from the local table (row e - ent_lo), the intact entity from hrows / trows, the relation
// from the replicated table.  The positive is scored on every rank from hrows / trows.
__device__ __forceinline__ RowPtrs shard_neg_rows(const MarginStepParams& a, long long w, long long ri,
                                                  bool head, long long loc) {
  const int np = ent_planes(a.model);
  const Planes<const float> e = table_planes(a.tb.ent0, a.tb.ent1, np, (size_t)loc * a.dim);
  const Planes<const float> h = head ? e : buf_planes(a.hrows, np, a.dim, w);
  const Planes<const float> t = head ? buf_planes(a.trows, np, a.dim, w) : e;
  return rows_of(h, t, rel_planes(a.model, a.dim, a.tb.rel0, a.tb.rel1, ri));
}

__device__ __forceinline__ RowPtrs shard_pos_rows(const MarginStepParams& a, long long w, long long ri) {
  const int np = ent_planes(a.model);
  return rows_of(buf_planes(a.hrows, np, a.dim, w), buf_planes(a.trows, np, a.dim, w),
                 rel_planes(a.model, a.dim, a.tb.rel0, a.tb.rel1, ri));
}

// An entity negative (draw_one, or draw_pos in a positional step): owned by the rank holding the drawn entity.
__device__ __forceinline__ bool owned_draw(const MarginStepParams& a, const PosCSR& pc, const PosSlices& ps,
                                           long long idx, float p_head, bool* head, long long* loc) {
  long long e;
  *head = pc.head_offs ? draw_pos(a.seed, a.offset, (uint64_t)idx, p_head, a.n_ent, ps, &e)
                      : draw_one(a.seed, a.offset, (uint64_t)idx, p_head, a.n_ent, &e);
  *loc = e - a.ent_lo;
  return (unsigned long long)*loc < (unsigned long long)a.n_rows;
}

// Negative idx of positive w in a sharded step: its kind (NEG_*), its relation nr and, if this rank scores
// it, true with loc = the local row of its replaced entity.  A relation-corrupting negative (a.n_rel > 0)
// is scored by the rank that holds the positive's head: its h / t rows are hrows / trows[w], so its
// entity gradients land in grad_hrows / grad_trows, which the ranks sum like every other.
__device__ __forceinline__ bool owned_negative(const MarginStepParams& a, const PosCSR& pc, const PosSlices& ps,
                                               long long w, long long idx, float p_head, long long ri, int* kind,
                                               long long* loc, long long* nr) {
  *nr = ri;
  if (a.n_rel == 0) {
    bool head;
    const bool own = owned_draw(a, pc, ps, idx, p_head, &head, loc);
    *kind = head ? NEG_HEAD : NEG_TAIL;
    return own;
  }
  long long e;
  *kind = draw_rel(a.seed, a.offset, (uint64_t)idx, p_head, a.rel_share, a.n_ent, a.n_rel, &e);
  if (*kind == NEG_REL) *nr = e;
  *loc = (*kind == NEG_REL ? a.h[w] : e) - a.ent_lo;
  return (unsigned long long)*loc < (unsigned long long)a.n_rows;
}

__device__ __forceinline__ RowPtrs shard_kind_rows(const MarginStepParams& a, long long w, long long nr, int kind,
                                                   long long loc) {
  return kind == NEG_REL ? shard_pos_rows(a, w, nr) : shard_neg_rows(a, w, nr, kind == NEG_HEAD, loc);
}

__global__ void margin_step_shard_fwd_kernel(MarginStepParams a, PosCSR pc) {
  const long long w = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= a.b) return;
  const long long ri = a.r[w];
  const float pos = triple_score(a.model, a.dim, shard_pos_rows(a, w, ri), lane, nullptr, nullptr);
  const float p_head = a.probs[ri];
  const PosSlices ps = generic_slices(pc, ri);
  float loss = 0.f;
  for (int j = 0; j < a.n_neg; ++j) {
    int kind;
    long long loc, nr;
    if (!owned_negative(a, pc, ps, w, (long long)j * a.b + w, p_head, ri, &kind, &loc, &nr)) continue;
    const float neg = triple_score(a.model, a.dim, shard_kind_rows(a, w, nr, kind, loc), lane, nullptr, nullptr);
    if (lane == 0) loss += pair_loss_term(a.loss_kind, a.margin, pos, neg);
  }
  if (lane == 0) atomicAdd(a.loss, loss);
}

// Backward of the sharded step: the replaced row's gradient goes to the local table (this rank owns
// it), the intact entity's and the positive's to grad_hrows / grad_trows[w], the relation's to the
// local copy of the relation gradient; the caller sums the last three over the ranks.  The positive's
// term is summed over the negatives this rank owns only, so the ranks' sums make up the whole.
__global__ void margin_step_shard_bwd_kernel(MarginStepParams a, TrainGrads gr, const float* gloss, PosCSR pc) {
  const long long w = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= a.b) return;
  const float g = *gloss;
  const long long ri = a.r[w];
  const RowPtrs pp = shard_pos_rows(a, w, ri);
  const float pos = triple_score(a.model, a.dim, pp, lane, nullptr, nullptr);
  const float p_head = a.probs[ri];
  const PosSlices ps = generic_slices(pc, ri);
  const int np = ent_planes(a.model);
  const Planes<float> gh = buf_planes(a.grad_hrows, np, a.dim, w);
  const Planes<float> gt = buf_planes(a.grad_trows, np, a.dim, w);
  const Planes<float> grel = rel_planes(a.model, a.dim, gr.rel0, gr.rel1, ri);
  double gpos_sum = 0.0;   // as in margin_step_bwd_kernel
  for (int j = 0; j < a.n_neg; ++j) {
    int kind;
    long long loc, nr;
    if (!owned_negative(a, pc, ps, w, (long long)j * a.b + w, p_head, ri, &kind, &loc, &nr)) continue;
    const RowPtrs pn = shard_kind_rows(a, w, nr, kind, loc);
    const float neg = triple_score(a.model, a.dim, pn, lane, nullptr, nullptr);
    float gp, gn;
    pair_loss_grads(a.loss_kind, a.margin, 1.f, pos, neg, &gp, &gn);
    gpos_sum += gp;
    if (kind == NEG_REL) {
      triple_backward(a.model, a.dim, pn, rows_of(gh, gt, rel_planes(a.model, a.dim, gr.rel0, gr.rel1, nr)), g * gn,
                      lane);
      continue;
    }
    const bool head = kind == NEG_HEAD;
    const Planes<float> ge = table_planes(gr.ent0, gr.ent1, np, (size_t)loc * a.dim);
    triple_backward(a.model, a.dim, pn, rows_of(head ? ge : gh, head ? gt : ge, grel), g * gn, lane);
  }
  triple_backward(a.model, a.dim, pp, rows_of(gh, gt, grel), g * (float)gpos_sum, lane);
}

// ------------------------------------------------------------------------------------------
// Fast fused step for the single-plane normalising models with a closed form per negative
// (TransE-L1 / TransE-L2 / DistMult), dim % 4 == 0, dim <= 256.
//
// One warp per positive triple.  Lane l owns the 16-byte chunks l and l + 32 of every row, so a
// row is two coalesced LDG.128 per lane (and two float4 atomics on the way back).  The positive's
// h, t, r rows are read ONCE and kept in registers as
//     A  = what a tail-corrupted negative is scored against  (DistMult: hn*r,  TransE: hn + r)
//     Bv = what a head-corrupted negative is scored against  (DistMult: r*tn,  TransE: tn - r)
// so each negative costs exactly one random row: its squared norm and its product with A / Bv
// come out of ONE two-value shuffle tree (TransE-L2 expands |P - en|^2 = |P|^2 - 2 P.en + |en|^2).
// Backward: the corrupted row's gradient is scattered immediately (the only unavoidable
// read-modify-write, 4*dim bytes per negative); the gradients of the intact entity and of the
// relation are linear in  V = sum over active negatives of en  (TransE-L1: of sign(P - en)),
// which stays in registers, so the positive's three rows are written once per positive instead of
// once per negative (the relation rows are shared by thousands of triples: 256x fewer atomics on
// the hottest addresses).
// Algorithmic traffic per positive: forward (n_neg + 3) * 4 dim bytes, backward the same rows
// again (recomputed, not stored) plus one RMW of each (SURVEY.md section 8d).
//
// That arithmetic is stated once, in fast_positive / fast_negative / fast_negative_backward /
// fast_positive_backward below, with the relation kind in fast_rel_negative / fast_rel_negative_backward
// (both_replaced_pair is the one case outside the closed form).  Two
// kernels run it, margin_step_fast_kernel and margin_step_ring_kernel: they differ only in how a
// negative's identity and row reach the warp, and that is all their bodies contain.
// ------------------------------------------------------------------------------------------
constexpr int FAST_NCH = 2;         // float4 chunks per lane
constexpr int FAST_MAX_DIM = 4 * 32 * FAST_NCH;

struct Vec { float4 c[FAST_NCH]; };

__device__ __forceinline__ Vec vec_load(const float* __restrict__ row, int dim, int lane) {
  Vec v;
#pragma unroll
  for (int i = 0; i < FAST_NCH; ++i) {
    const int k = 4 * (lane + 32 * i);
    v.c[i] = k < dim ? __ldg(reinterpret_cast<const float4*>(row + k)) : make_float4(0.f, 0.f, 0.f, 0.f);
  }
  return v;
}
__device__ __forceinline__ void vec_atomic_add(float* __restrict__ row, int dim, int lane, const Vec& v) {
#pragma unroll
  for (int i = 0; i < FAST_NCH; ++i) {
    const int k = 4 * (lane + 32 * i);
    if (k < dim) atomicAdd(reinterpret_cast<float4*>(row + k), v.c[i]);
  }
}
template <class F>
__device__ __forceinline__ Vec vec_map(const Vec& a, const Vec& b, F f) {
  Vec o;
#pragma unroll
  for (int i = 0; i < FAST_NCH; ++i)
    o.c[i] = make_float4(f(a.c[i].x, b.c[i].x), f(a.c[i].y, b.c[i].y), f(a.c[i].z, b.c[i].z),
                         f(a.c[i].w, b.c[i].w));
  return o;
}
template <class F>
__device__ __forceinline__ Vec vec_map3(const Vec& a, const Vec& b, const Vec& c, F f) {
  Vec o;
#pragma unroll
  for (int i = 0; i < FAST_NCH; ++i)
    o.c[i] = make_float4(f(a.c[i].x, b.c[i].x, c.c[i].x), f(a.c[i].y, b.c[i].y, c.c[i].y),
                         f(a.c[i].z, b.c[i].z, c.c[i].z), f(a.c[i].w, b.c[i].w, c.c[i].w));
  return o;
}
__device__ __forceinline__ Vec vec_scale(const Vec& a, float s) {
  return vec_map(a, a, [s](float x, float) { return x * s; });
}
__device__ __forceinline__ float vec_dot(const Vec& a, const Vec& b) {
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < FAST_NCH; ++i) {
    s = fmaf(a.c[i].x, b.c[i].x, s); s = fmaf(a.c[i].y, b.c[i].y, s);
    s = fmaf(a.c[i].z, b.c[i].z, s); s = fmaf(a.c[i].w, b.c[i].w, s);
  }
  return s;
}
__device__ __forceinline__ float vec_l1_diff(const Vec& a, const Vec& b) {
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < FAST_NCH; ++i)
    s += fabsf(a.c[i].x - b.c[i].x) + fabsf(a.c[i].y - b.c[i].y) + fabsf(a.c[i].z - b.c[i].z) +
         fabsf(a.c[i].w - b.c[i].w);
  return s;
}
__device__ __forceinline__ void warp_sum2(float& a, float& b) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    a += __shfl_xor_sync(0xffffffffu, a, o);
    b += __shfl_xor_sync(0xffffffffu, b, o);
  }
}
__device__ __forceinline__ float sgn(float x) { return x > 0.f ? 1.f : (x < 0.f ? -1.f : 0.f); }

// The positive, as its negatives see it.
struct FastPos {
  Vec r, hn, tn;       // the relation's row; the normalised head and tail
  float inv_h, inv_t;  // 1 / max(|h|, eps), 1 / max(|t|, eps)
  float sA, sB;        // |A|^2, |Bv|^2 (TransE-L2)
  float pos;           // its score
};
// A and Bv are an object of their own: a negative picks one of them by address (head ? Bv : A), and the
// compiler keeps the whole object addressed that way in local memory.  As members of FastPos they take
// the positive's other rows there with them (192 stack bytes instead of these 64).
struct FastAB { Vec A, Bv; };

// hrow / trow / rrow: the positive's three rows in global memory, read here and nowhere else.
template <int MODEL>
__device__ __forceinline__ void fast_positive(const float* hrow, const float* trow, const float* rrow, int dim,
                                              int lane, FastPos& p, FastAB& ab) {
  const Vec h = vec_load(hrow, dim, lane);
  const Vec t = vec_load(trow, dim, lane);
  p.r = vec_load(rrow, dim, lane);
  float sh = vec_dot(h, h), stt = vec_dot(t, t);
  warp_sum2(sh, stt);
  p.inv_h = 1.0f / fmaxf(sqrtf(sh), NORM_EPS);
  p.inv_t = 1.0f / fmaxf(sqrtf(stt), NORM_EPS);
  p.hn = vec_scale(h, p.inv_h);
  p.tn = vec_scale(t, p.inv_t);
  if constexpr (MODEL == KGE_DISTMULT) {
    ab.A = vec_map(p.hn, p.r, [](float x, float y) { return x * y; });
    ab.Bv = vec_map(p.r, p.tn, [](float x, float y) { return x * y; });
  } else {
    ab.A = vec_map(p.hn, p.r, [](float x, float y) { return x + y; });
    ab.Bv = vec_map(p.tn, p.r, [](float x, float y) { return x - y; });
  }
  p.sA = p.sB = 0.f;
  if constexpr (MODEL == KGE_DISTMULT) {
    p.pos = warp_sum(vec_dot(ab.A, p.tn));
  } else if constexpr (MODEL == KGE_TRANSE_L2) {
    p.sA = vec_dot(ab.A, ab.A); p.sB = vec_dot(ab.Bv, ab.Bv);
    warp_sum2(p.sA, p.sB);
    const Vec x = vec_map(ab.A, p.tn, [](float a_, float q) { return a_ - q; });
    p.pos = -warp_sum(vec_dot(x, x));
  } else {
    p.pos = -warp_sum(vec_l1_diff(ab.A, p.tn));
  }
}

// One negative, scored from its corrupted entity's row ev (head: the head is the replaced end).
struct FastNeg {
  float neg, inv_e;  // its score; 1 / max(|e|, eps)
  float en_dot_G;    // en . (d neg / d en), needed by the normalisation Jacobian
  Vec en;            // the normalised row: TransE-L1 scores with it, the others need it in the backward only
};

template <int MODEL, bool BWD>
__device__ __forceinline__ void fast_negative(const FastPos& p, const FastAB& ab, const Vec& ev, bool head,
                                              FastNeg& n) {
  const Vec& P = head ? ab.Bv : ab.A;
  float se = vec_dot(ev, ev), sp = vec_dot(ev, P);
  warp_sum2(se, sp);
  n.inv_e = 1.0f / fmaxf(sqrtf(se), NORM_EPS);
  n.en_dot_G = 0.f;
  if constexpr (MODEL == KGE_DISTMULT) {
    n.neg = sp * n.inv_e;
    n.en_dot_G = n.neg;
  } else if constexpr (MODEL == KGE_TRANSE_L2) {
    const float sP = head ? p.sB : p.sA;
    const float ee = n.inv_e * n.inv_e * se, pe = n.inv_e * sp;
    n.neg = -(sP - 2.f * pe + ee);
    n.en_dot_G = 2.f * (pe - ee);
  } else {
    n.en = vec_scale(ev, n.inv_e);
    float l1 = vec_l1_diff(P, n.en), eg = 0.f;
    if (BWD) {
      const Vec sg = vec_map(P, n.en, [](float a_, float q) { return sgn(a_ - q); });
      eg = vec_dot(n.en, sg);
    }
    warp_sum2(l1, eg);
    n.neg = -l1;
    n.en_dot_G = eg;
  }
}

// Lane 0 keeps the loss term of the pair (pos, neg); the forward writes the negative's score out.
template <bool BWD, int LOSS>
__device__ __forceinline__ void pair_forward(const MarginStepParams& a, long long idx, int lane, float pos,
                                             float neg, float& loss) {
  const float term = pair_loss_term(LOSS, a.margin, pos, neg);
  if (lane == 0) {
    if (!BWD && a.neg_out) a.neg_out[idx] = neg;
    loss += term;
  }
}

// What the backward sums over one positive's negatives.  The closed form is linear in the negatives, so
// a loss other than the margin only turns the counts into weights: negative j enters V, its kind's sum
// and its own scatter with weight c_j = dl/dneg_j, and the positive with -sum_j dl/dpos instead of the
// active count.  For the margin loss c_j = 1 on every active hinge and the weights drop out at compile
// time.  The weights and dl/dpos are non-integers summed over up to thousands of negatives: in double, as
// fp32 would drift by ~n eps.
template <int LOSS>
struct FastAcc {
  using Count = std::conditional_t<LOSS == KGE_LOSS_MARGIN, int, double>;
  Vec Vt, Vh;              // V over the tail- / head-corrupted negatives
  Count n_t = 0, n_h = 0;  // per kind: the active hinges (margin) or the summed weights c_j
  double gpos_sum = 0.0;   // LOSS != margin: sum of dl/dpos
  __device__ __forceinline__ FastAcc() {
#pragma unroll
    for (int i = 0; i < FAST_NCH; ++i) Vt.c[i] = Vh.c[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
};

// Backward of one negative: its row's gradient, g c_j (G - en (en . G)) * inv_e with G = d neg / d en,
// goes to dst at once; c_j V and c_j go into acc.
template <int MODEL, int LOSS>
__device__ __forceinline__ void fast_negative_backward(const FastPos& p, const FastAB& ab, const Vec& ev, bool head,
                                                       const FastNeg& n, float margin, float g, float* dst,
                                                       int dim, int lane, FastAcc<LOSS>& acc) {
  float gp, cj;   // dl/dpos and dl/dneg of this pair (g = 1)
  pair_loss_grads(LOSS, margin, 1.f, p.pos, n.neg, &gp, &cj);
  if constexpr (LOSS != KGE_LOSS_MARGIN) acc.gpos_sum += gp;
  if (cj == 0.f) return;
  const float wj = LOSS == KGE_LOSS_MARGIN ? 1.f : cj;
  const Vec& P = head ? ab.Bv : ab.A;
  Vec en;
  if constexpr (MODEL == KGE_TRANSE_L1) en = n.en;
  else en = vec_scale(ev, n.inv_e);
  const float en_dot_G = n.en_dot_G;
  Vec ge, V;
  const float c = LOSS == KGE_LOSS_MARGIN ? g * n.inv_e : g * wj * n.inv_e;
  if constexpr (MODEL == KGE_DISTMULT) {
    ge = vec_map(P, en, [=](float a_, float q) { return c * (a_ - q * en_dot_G); });
    V = LOSS == KGE_LOSS_MARGIN ? en : vec_scale(en, wj);
  } else if constexpr (MODEL == KGE_TRANSE_L2) {
    ge = vec_map(P, en, [=](float a_, float q) { return c * (2.f * (a_ - q) - q * en_dot_G); });
    V = LOSS == KGE_LOSS_MARGIN ? en : vec_scale(en, wj);
  } else {
    V = vec_map(P, en, [](float a_, float q) { return sgn(a_ - q); });
    ge = vec_map(V, en, [=](float s_, float q) { return c * (s_ - q * en_dot_G); });
    if constexpr (LOSS != KGE_LOSS_MARGIN) V = vec_scale(V, wj);
  }
  vec_atomic_add(dst, dim, lane, ge);
  using Count = typename FastAcc<LOSS>::Count;
  const Count inc = LOSS == KGE_LOSS_MARGIN ? Count(1) : Count(wj);
  if (head) { acc.Vh = vec_map(acc.Vh, V, [](float x, float y) { return x + y; }); acc.n_h += inc; }
  else { acc.Vt = vec_map(acc.Vt, V, [](float x, float y) { return x + y; }); acc.n_t += inc; }
}

// The relation kind (BernoulliRelationNegativeSampler): a negative (h, t, r') keeps the positive's entities,
// so it is scored from its relation row r' against C, a function of the positive's hn and tn alone:
//     DistMult: neg = C . r',  C = hn * tn        TransE: neg = -|C + r'|,  C = hn - tn
// (TransE-L2 expands |C + r'|^2 = |C|^2 + 2 C.r' + |r'|^2).  C costs a few lane-local flops, so it is formed
// where it is used rather than held next to A and Bv.  The relation row is not normalised.
template <int MODEL>
__device__ __forceinline__ Vec rel_C(const FastPos& p) {
  if constexpr (MODEL == KGE_DISTMULT) return vec_map(p.hn, p.tn, [](float x, float y) { return x * y; });
  else return vec_map(p.hn, p.tn, [](float x, float y) { return x - y; });
}

// What the backward sums over the relation negatives: W = sum_j c_j r'_j (TransE-L1: of c_j sign(C + r'_j))
// and their summed weights.  The positive's hn / tn gradients from them are linear in W (and n_r).
template <int LOSS>
struct FastRelAcc {
  using Count = typename FastAcc<LOSS>::Count;
  Vec W;
  Count n_r = 0;
  float sC = 0.f;          // |C|^2 (TransE-L2), set with the positive
  __device__ __forceinline__ FastRelAcc() {
#pragma unroll
    for (int i = 0; i < FAST_NCH; ++i) W.c[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
};

template <int MODEL, int LOSS>
__device__ __forceinline__ void fast_rel_positive(const FastPos& p, FastRelAcc<LOSS>& rl) {
  if constexpr (MODEL == KGE_TRANSE_L2) {
    const Vec C = rel_C<MODEL>(p);
    rl.sC = warp_sum(vec_dot(C, C));
  }
}

// One relation negative, scored from its relation row rv.
template <int MODEL, int LOSS>
__device__ __forceinline__ void fast_rel_negative(const FastPos& p, const FastRelAcc<LOSS>& rl, const Vec& rv,
                                                  FastNeg& n) {
  const Vec C = rel_C<MODEL>(p);
  n.inv_e = 1.f;
  n.en_dot_G = 0.f;
  if constexpr (MODEL == KGE_DISTMULT) {
    n.neg = warp_sum(vec_dot(C, rv));
  } else if constexpr (MODEL == KGE_TRANSE_L2) {
    float se = vec_dot(rv, rv), sp = vec_dot(rv, C);
    warp_sum2(se, sp);
    n.neg = -(rl.sC + 2.f * sp + se);
  } else {
    n.neg = -warp_sum(vec_l1_diff(C, vec_scale(rv, -1.f)));
  }
}

// Backward of one relation negative: g c_j d neg / d r' goes to its relation row dst at once; c_j r'_j
// (TransE-L1: c_j sign(C + r'_j)) and c_j go into rl, dl/dpos into acc.
template <int MODEL, int LOSS>
__device__ __forceinline__ void fast_rel_negative_backward(const FastPos& p, const Vec& rv, const FastNeg& n,
                                                           float margin, float g, float* dst, int dim, int lane,
                                                           FastAcc<LOSS>& acc, FastRelAcc<LOSS>& rl) {
  float gp, cj;
  pair_loss_grads(LOSS, margin, 1.f, p.pos, n.neg, &gp, &cj);
  if constexpr (LOSS != KGE_LOSS_MARGIN) acc.gpos_sum += gp;
  if (cj == 0.f) return;
  const float wj = LOSS == KGE_LOSS_MARGIN ? 1.f : cj;
  const float c = g * wj;
  const Vec C = rel_C<MODEL>(p);
  Vec gr, V;
  if constexpr (MODEL == KGE_DISTMULT) {
    gr = vec_scale(C, c);
    V = LOSS == KGE_LOSS_MARGIN ? rv : vec_scale(rv, wj);
  } else if constexpr (MODEL == KGE_TRANSE_L2) {
    gr = vec_map(C, rv, [=](float a_, float q) { return -2.f * c * (a_ + q); });
    V = LOSS == KGE_LOSS_MARGIN ? rv : vec_scale(rv, wj);
  } else {
    const Vec sg = vec_map(C, rv, [](float a_, float q) { return sgn(a_ + q); });
    gr = vec_scale(sg, -c);
    V = LOSS == KGE_LOSS_MARGIN ? sg : vec_scale(sg, wj);
  }
  vec_atomic_add(dst, dim, lane, gr);
  using Count = typename FastAcc<LOSS>::Count;
  rl.W = vec_map(rl.W, V, [](float x, float y) { return x + y; });
  rl.n_r += LOSS == KGE_LOSS_MARGIN ? Count(1) : Count(wj);
}

// Backward of the positive, once: gradients with respect to hn, tn, r (+g c_j per negative, -g fn for
// the positive), through the normalisation, added into the three destination rows.  REL: the relation
// negatives' hn / tn terms too, from rl.
template <int MODEL, int LOSS, bool REL = false>
__device__ __forceinline__ void fast_positive_backward(const FastPos& p, const FastAB& ab, const FastAcc<LOSS>& acc,
                                                       float g, float* dst_h, float* dst_t, float* dst_r,
                                                       int dim, int lane, const FastRelAcc<LOSS>* rl = nullptr) {
  using Count = typename FastAcc<LOSS>::Count;
  Count n_r = 0;
  if constexpr (REL) n_r = rl->n_r;
  if constexpr (LOSS == KGE_LOSS_MARGIN) {
    if (acc.n_t + acc.n_h + n_r == 0) return;
  } else {
    if (acc.n_t == 0.0 && acc.n_h == 0.0 && n_r == 0.0 && acc.gpos_sum == 0.0) return;
  }
  // fn: the positive's weight, -sum_j dl/dpos (the margin loss: the active count)
  const float fn_t = (float)acc.n_t, fn_h = (float)acc.n_h;
  const float fn = LOSS == KGE_LOSS_MARGIN ? (float)(acc.n_t + acc.n_h + n_r) : (float)-acc.gpos_sum;
  const Vec& Vt = acc.Vt;
  const Vec& Vh = acc.Vh;
  Vec Gh, Gt, Gr;
  if constexpr (MODEL == KGE_DISTMULT) {
    // neg_t = sum A en, A = hn r ;  neg_h = sum en Bv, Bv = r tn ;  pos = sum hn r tn
    Gh = vec_map3(p.r, Vt, p.tn, [=](float rr, float vt, float tt) { return g * rr * (vt - fn * tt); });
    Gt = vec_map3(p.r, Vh, p.hn, [=](float rr, float vh, float hh) { return g * rr * (vh - fn * hh); });
    const Vec tmp = vec_map3(p.hn, Vt, p.tn, [=](float hh, float vt, float tt) { return hh * (vt - fn * tt); });
    Gr = vec_map3(tmp, p.tn, Vh, [=](float x, float tt, float vh) { return g * (x + tt * vh); });
  } else if constexpr (MODEL == KGE_TRANSE_L2) {
    // neg_t = -|A - en|^2 ; neg_h = -|en - Bv|^2 ; pos = -|x|^2, x = A - tn
    const Vec x = vec_map(ab.A, p.tn, [](float a_, float q) { return a_ - q; });
    const Vec dt = vec_map3(ab.A, Vt, x, [=](float aa, float vt, float xx) {  // sum_t (A - en) - n x
      return fn_t * aa - vt - fn * xx; });
    const Vec dh = vec_map(Vh, ab.Bv, [=](float vh, float bb) { return vh - fn_h * bb; });  // sum_h (en - Bv)
    Gh = vec_scale(dt, -2.f * g);
    Gt = vec_map3(dh, x, x, [=](float d, float xx, float) { return 2.f * g * (d - fn * xx); });
    Gr = vec_map(dt, dh, [=](float a_, float q) { return -2.f * g * (a_ + q); });
  } else {
    // neg_t = -|A - en|_1 (V = sign(A - en)) ; neg_h = -|Bv - en|_1 (V = sign(Bv - en)) ; pos = -|x|_1
    const Vec sx = vec_map(ab.A, p.tn, [](float a_, float q) { return sgn(a_ - q); });
    Gh = vec_map(Vt, sx, [=](float vt, float s_) { return g * (fn * s_ - vt); });
    Gt = vec_map(Vh, sx, [=](float vh, float s_) { return g * (-vh - fn * s_); });
    Gr = vec_map3(Vt, Vh, sx, [=](float vt, float vh, float s_) { return g * (vh - vt + fn * s_); });
  }
  if constexpr (REL) {
    // relation negatives: d neg / d hn = tn r' (DistMult), -2 (C + r') (TransE-L2), -sign(C + r') (L1);
    // d neg / d tn the same with hn for tn (DistMult) or the opposite sign (TransE)
    const Vec& W = rl->W;
    Vec Q;
    if constexpr (MODEL == KGE_DISTMULT) {
      Q = W;
    } else if constexpr (MODEL == KGE_TRANSE_L2) {
      const float fr = (float)n_r;
      Q = vec_map(rel_C<MODEL>(p), W, [=](float cc, float w_) { return -2.f * (fr * cc + w_); });
    } else {
      Q = vec_scale(W, -1.f);
    }
    if constexpr (MODEL == KGE_DISTMULT) {
      Gh = vec_map3(Gh, p.tn, Q, [=](float a_, float tt, float q) { return a_ + g * tt * q; });
      Gt = vec_map3(Gt, p.hn, Q, [=](float a_, float hh, float q) { return a_ + g * hh * q; });
    } else {
      Gh = vec_map(Gh, Q, [=](float a_, float q) { return a_ + g * q; });
      Gt = vec_map(Gt, Q, [=](float a_, float q) { return a_ - g * q; });
    }
  }
  float ph = vec_dot(p.hn, Gh), pt = vec_dot(p.tn, Gt);
  warp_sum2(ph, pt);
  const float inv_h = p.inv_h, inv_t = p.inv_t;
  const Vec gh = vec_map(Gh, p.hn, [=](float gg, float q) { return (gg - q * ph) * inv_h; });
  const Vec gt = vec_map(Gt, p.tn, [=](float gg, float q) { return (gg - q * pt) * inv_t; });
  vec_atomic_add(dst_h, dim, lane, gh);
  vec_atomic_add(dst_t, dim, lane, gt);
  vec_atomic_add(dst_r, dim, lane, Gr);
}

// A negative with more than one position replaced (possible with caller-supplied negatives only) is outside
// the closed form: the generic score, and in the backward the generic gradients of the negative and of
// the positive for this pair alone.
template <int MODEL, bool BWD, int LOSS>
__device__ __forceinline__ void both_replaced_pair(const MarginStepParams& a, const TrainGrads& gr, long long hi,
                                                   long long ti, long long ri, long long nh, long long nt,
                                                   long long idx, float pos, float g, int lane, float& loss,
                                                   long long nr) {
  const RowPtrs pn = table_rows(MODEL, a.dim, a.tb, nh, nt, nr);
  const float neg = triple_score(MODEL, a.dim, pn, lane, nullptr, nullptr);
  pair_forward<BWD, LOSS>(a, idx, lane, pos, neg, loss);
  if constexpr (BWD) {
    float gp, gn;   // g = 1; the margin loss: -1 and 1 on an active hinge
    pair_loss_grads(LOSS, a.margin, 1.f, pos, neg, &gp, &gn);
    if (gn != 0.f || gp != 0.f) {
      triple_backward(MODEL, a.dim, pn, table_rows(MODEL, a.dim, gr, nh, nt, nr),
                      LOSS == KGE_LOSS_MARGIN ? g : g * gn, lane);
      const RowPtrs pp = table_rows(MODEL, a.dim, a.tb, hi, ti, ri);
      triple_backward(MODEL, a.dim, pp, table_rows(MODEL, a.dim, gr, hi, ti, ri),
                      LOSS == KGE_LOSS_MARGIN ? -g : g * gp, lane);
    }
  }
}

// Register-resident form: no shared memory.  Philox draws are made 32 negatives at a time, one per
// lane, and handed round by shuffle; PF rows at a time are loaded into registers and then reduced.
// Margin loss only (launch_margin_step): the other losses take the ring or the generic kernels.
template <int MODEL, bool BWD>
__global__ void __launch_bounds__(WARPS_PER_BLOCK * 32, 4)
margin_step_fast_kernel(MarginStepParams a, TrainGrads gr, const float* __restrict__ gloss) {
  constexpr int PF = BWD ? 2 : 4;  // negatives whose rows are in flight together, per warp
  constexpr int LOSS = KGE_LOSS_MARGIN;
  const long long w = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= a.b) return;
  const int dim = a.dim;
  const float* __restrict__ ent = a.tb.ent0;
  const long long hi = a.h[w], ti = a.t[w], ri = a.r[w];
  FastPos pp;
  FastAB ab;
  fast_positive<MODEL>(ent + (size_t)hi * dim, ent + (size_t)ti * dim, a.tb.rel0 + (size_t)ri * dim, dim, lane, pp,
                       ab);
  if (lane == 0 && a.pos_out && !BWD) a.pos_out[w] = pp.pos;
  const float p_head = a.nh ? 0.f : a.probs[ri];
  const float g = BWD ? *gloss : 0.f;
  float loss = 0.f;
  FastAcc<LOSS> acc;
  for (int j0 = 0; j0 < a.n_neg; j0 += 32) {
    // this lane's draw for negative j0 + lane
    long long my_nh = hi, my_nt = ti;
    if (j0 + lane < a.n_neg) {
      const long long idx = (long long)(j0 + lane) * a.b + w;
      if (a.nh) { my_nh = a.nh[idx]; my_nt = a.nt[idx]; }
      else corrupt_one(a.seed, a.offset, (uint64_t)idx, p_head, a.n_ent, hi, ti, &my_nh, &my_nt);
      if (!BWD && a.nh_out) { a.nh_out[idx] = my_nh; a.nt_out[idx] = my_nt; }
    }
    const int jn = min(32, a.n_neg - j0);
    // PF negatives at a time: their rows are requested together (memory-level parallelism:
    // PF x 4 dim bytes in flight per warp), then reduced one after the other
    for (int jj0 = 0; jj0 < jn; jj0 += PF) {
      long long nhs[PF], nts[PF];
      Vec evs[PF];
#pragma unroll
      for (int u = 0; u < PF; ++u) {
        const int jj = min(jj0 + u, 31);
        nhs[u] = __shfl_sync(0xffffffffu, my_nh, jj);
        nts[u] = __shfl_sync(0xffffffffu, my_nt, jj);
        const bool both = nhs[u] != hi && nts[u] != ti;
        const long long e_ = nhs[u] != hi ? nhs[u] : nts[u];
        if (jj0 + u < jn && !both) evs[u] = vec_load(ent + (size_t)e_ * dim, dim, lane);
      }
#pragma unroll
      for (int u = 0; u < PF; ++u) {
        if (jj0 + u >= jn) break;
        const long long nh = nhs[u], nt = nts[u];
        const long long idx = (long long)(j0 + jj0 + u) * a.b + w;
        if (nh != hi && nt != ti) {
          both_replaced_pair<MODEL, BWD, LOSS>(a, gr, hi, ti, ri, nh, nt, idx, pp.pos, g, lane, loss, ri);
          continue;
        }
        const bool head = nh != hi;            // warp-uniform
        FastNeg n;
        fast_negative<MODEL, BWD>(pp, ab, evs[u], head, n);
        pair_forward<BWD, LOSS>(a, idx, lane, pp.pos, n.neg, loss);
        if constexpr (BWD)
          fast_negative_backward<MODEL, LOSS>(pp, ab, evs[u], head, n, a.margin, g,
                                              gr.ent0 + (size_t)(head ? nh : nt) * dim, dim, lane, acc);
      }
    }
  }
  if constexpr (BWD)
    fast_positive_backward<MODEL, LOSS>(pp, ab, acc, g, gr.ent0 + (size_t)hi * dim, gr.ent0 + (size_t)ti * dim,
                                        gr.rel0 + (size_t)ri * dim, dim, lane);
  else if (lane == 0) atomicAdd(a.loss, loss);
}

// ------------------------------------------------------------------------------------------
// Ring variant of the fast fused step: the corrupted entities' rows travel through a per-warp
// shared-memory ring filled by 1-D bulk async copies (cp.async.bulk, completion on an mbarrier per
// slot) instead of through registers.  The register form keeps PF = 4 (2 backward) rows in flight
// per warp and stalls on them before every reduction -- measured 0.53 of the HBM copy bandwidth
// with 16 resident warps per SM (ncu: warps active 24 %).  Here a warp keeps RING rows in flight
// at all times (8 x 800 B = 6.4 KB), independently of its register budget, the Philox draws of all
// negatives are made up front into shared memory, and row j + RING is requested the moment row j
// has been consumed.  The arithmetic per negative is the closed form stated above.
// Shared memory per warp: RING * row_bytes + 4 * n_neg (codes) + RING barriers.
// ------------------------------------------------------------------------------------------
constexpr int RING = 8;
constexpr unsigned CODE_BOTH = 0xFFFFFFFFu;   // caller-supplied negative with both ends replaced

__device__ __forceinline__ Vec vec_load_smem(const float* row, int dim, int lane) {
  Vec v;
#pragma unroll
  for (int i = 0; i < FAST_NCH; ++i) {
    const int k = 4 * (lane + 32 * i);
    v.c[i] = k < dim ? *reinterpret_cast<const float4*>(row + k) : make_float4(0.f, 0.f, 0.f, 0.f);
  }
  return v;
}

// MINB: minimum resident CTAs per SM the register allocation is held to (0: the compiler's choice --
// 72 registers forward, 128 backward; 5 holds the backward form to 96 registers, 20 warps per SM)
// SHARD: the entity-sharded step (MarginStepParams::hrows).  The positive's h / t come from hrows /
// trows, the draw loop keeps only the negatives whose replaced entity this rank holds (ballot +
// prefix, local row numbers in `codes`), so the ring streams owned rows only, and the positive's
// gradients go to grad_hrows / grad_trows[w].
// LOSS: KGE_LOSS_*; it turns the backward's counts into weights (FastAcc).
// REL: the relation-corrupting step (a.n_rel > 0, margin_step_ring_rel_kernel).  A relation negative's
// code carries CODE_REL and its relation; its row streams through the same ring from the relation table.
// SHARD: the rank holding the positive's head scores it.  Codes then hold 30-bit row numbers.
// POS: the positional step (pc, margin_step_ring_pos_kernel): entity negatives from draw_pos,
// whose two candidate slices the warp loads once, since all its negatives share the positive's relation.
constexpr unsigned CODE_REL = 0x40000000u;

template <int MODEL, bool BWD, bool SHARD, int LOSS, bool REL, bool POS = false>
__device__ __forceinline__ void ring_step(const MarginStepParams& a, const TrainGrads& gr, const float* gloss,
                                          const PosCSR& pc = PosCSR{}) {
  extern __shared__ __align__(128) unsigned char ring_smem[];
  const int warp_in_block = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long w = (long long)blockIdx.x * WARPS_PER_BLOCK + warp_in_block;
  const int dim = a.dim;
  const unsigned row_bytes = (unsigned)dim * 4u;                 // dim % 4 == 0: a multiple of 16
  const int n_codes = (a.n_neg + 3) & ~3;
  const size_t per_warp = (size_t)RING * row_bytes + (size_t)n_codes * 4 + RING * sizeof(uint64_t);
  unsigned char* base = ring_smem + (size_t)warp_in_block * ((per_warp + 127) & ~(size_t)127);
  float* ring = reinterpret_cast<float*>(base);
  unsigned* codes = reinterpret_cast<unsigned*>(base + (size_t)RING * row_bytes);
  uint64_t* bars = reinterpret_cast<uint64_t*>(base + (size_t)RING * row_bytes + (size_t)n_codes * 4);
  if (w >= a.b) return;          // whole warps only: no block-wide barrier below
  if (lane == 0) {
#pragma unroll
    for (int s_ = 0; s_ < RING; ++s_) ptx::mbar_init(&bars[s_], 1);
    ptx::fence_mbar_init();
  }
  const float* __restrict__ ent = a.tb.ent0;
  const long long hi = a.h[w], ti = a.t[w], ri = a.r[w];
  const float p_head = a.nh ? 0.f : a.probs[ri];
  constexpr unsigned ROW_MASK = REL ? 0x3FFFFFFFu : 0x7FFFFFFFu;
  PosSlices ps;
  if constexpr (POS) ps = pos_slices(pc, ri);
  // ---- all corruptions of this positive, up front: code = entity | head flag (REL: or relation | CODE_REL) ----
  int n_loop = a.n_neg;            // SHARD: the owned negatives, compacted to the front of `codes`
  if constexpr (SHARD) {
    n_loop = 0;
    const bool own_head = (unsigned long long)(hi - a.ent_lo) < (unsigned long long)a.n_rows;
    for (int j0 = 0; j0 < a.n_neg; j0 += 32) {
      const int j = j0 + lane;
      bool own = false;
      unsigned code = 0u;
      if (j < a.n_neg) {
        const uint64_t idx = (uint64_t)((long long)j * a.b + w);
        long long e;
        if constexpr (REL) {
          const int kind = draw_rel(a.seed, a.offset, idx, p_head, a.rel_share, a.n_ent, a.n_rel, &e);
          if (kind == NEG_REL) {
            own = own_head;
            code = (unsigned)e | CODE_REL;
          } else {
            const unsigned long long loc = (unsigned long long)(e - a.ent_lo);
            own = loc < (unsigned long long)a.n_rows;
            code = (unsigned)loc | (kind == NEG_HEAD ? 0x80000000u : 0u);
          }
        } else {
          bool head;
          if constexpr (POS) head = draw_pos(a.seed, a.offset, idx, p_head, a.n_ent, ps, &e);
          else head = draw_one(a.seed, a.offset, idx, p_head, a.n_ent, &e);
          const unsigned long long loc = (unsigned long long)(e - a.ent_lo);
          own = loc < (unsigned long long)a.n_rows;      // n_rows < 2^31 (ring_step_ok)
          code = (unsigned)loc | (head ? 0x80000000u : 0u);
        }
      }
      const unsigned ball = __ballot_sync(0xffffffffu, own);
      if (own) codes[n_loop + __popc(ball & ((1u << lane) - 1u))] = code;
      n_loop += __popc(ball);
    }
  } else {
    for (int j0 = 0; j0 < a.n_neg; j0 += 32) {
      const int j = j0 + lane;
      if (j < a.n_neg) {
        const long long idx = (long long)j * a.b + w;
        long long nh = hi, nt = ti;
        if constexpr (REL) {
          long long nr = ri;
          step_negative(a, idx, p_head, hi, ti, ri, &nh, &nt, &nr);
          if (!BWD && a.nh_out) { a.nh_out[idx] = nh; a.nt_out[idx] = nt; }
          if (!BWD && a.nr_out) a.nr_out[idx] = nr;
          const int changed = (nh != hi) + (nt != ti) + (nr != ri);
          const bool head = nh != hi;
          codes[j] = changed > 1 ? CODE_BOTH
                     : nr != ri ? ((unsigned)nr | CODE_REL)
                                : ((unsigned)(head ? nh : nt) | (head ? 0x80000000u : 0u));
        } else if constexpr (POS) {   // no caller negatives (kge_pos_step_*): one end is replaced
          long long e;
          const bool head = draw_pos(a.seed, a.offset, (uint64_t)idx, p_head, a.n_ent, ps, &e);
          if (!BWD && a.nh_out) { a.nh_out[idx] = head ? e : hi; a.nt_out[idx] = head ? ti : e; }
          codes[j] = (unsigned)e | (head ? 0x80000000u : 0u);
        } else {
          if (a.nh) { nh = a.nh[idx]; nt = a.nt[idx]; }
          else corrupt_one(a.seed, a.offset, (uint64_t)idx, p_head, a.n_ent, hi, ti, &nh, &nt);
          if (!BWD && a.nh_out) { a.nh_out[idx] = nh; a.nt_out[idx] = nt; }
          const bool head = nh != hi;
          codes[j] = (nh != hi && nt != ti) ? CODE_BOTH : ((unsigned)(head ? nh : nt) | (head ? 0x80000000u : 0u));
        }
      }
    }
  }
  __syncwarp();
  auto request = [&](int j) {      // lane 0: start the copy of negative j's row into its slot
    const unsigned code = codes[j];
    if (!SHARD && code == CODE_BOTH) return;
    const int slot = j % RING;
    const float* src = REL && (code & CODE_REL) ? a.tb.rel0 : ent;
    ptx::mbar_arrive_expect_tx(&bars[slot], row_bytes);
    ptx::bulk_g2s(ring + (size_t)slot * dim, src + (size_t)(code & ROW_MASK) * dim, row_bytes, &bars[slot]);
  };
  if (lane == 0) {
    const int first = n_loop < RING ? n_loop : RING;
    for (int j = 0; j < first; ++j) request(j);
  }
  // ---- the positive (its three rows come straight from global memory, once) ----
  FastPos pp;
  FastAB ab;
  fast_positive<MODEL>(SHARD ? a.hrows + (size_t)w * dim : ent + (size_t)hi * dim,
                       SHARD ? a.trows + (size_t)w * dim : ent + (size_t)ti * dim,
                       a.tb.rel0 + (size_t)ri * dim, dim, lane, pp, ab);
  if (lane == 0 && a.pos_out && !BWD) a.pos_out[w] = pp.pos;
  const float g = BWD ? *gloss : 0.f;
  float loss = 0.f;
  FastAcc<LOSS> acc;
  FastRelAcc<LOSS> rl;
  if constexpr (REL) fast_rel_positive<MODEL, LOSS>(pp, rl);
  unsigned phases = 0u;   // bit s = parity of the next completion of slot s (a skipped use does not advance it)
  for (int j = 0; j < n_loop; ++j) {
    const unsigned code = codes[j];
    const long long idx = (long long)j * a.b + w;   // (unsharded: the negative's index in nh / nt / neg_out)
    if (!SHARD && code == CODE_BOTH) {   // no ring slot
      both_replaced_pair<MODEL, BWD, LOSS>(a, gr, hi, ti, ri, a.nh[idx], a.nt[idx], idx, pp.pos, g, lane, loss,
                                           REL ? a.nr[idx] : ri);
      if (lane == 0 && j + RING < n_loop) request(j + RING);
      continue;
    }
    const int slot = j % RING;
    ptx::mbar_wait(&bars[slot], (phases >> slot) & 1u);
    phases ^= 1u << slot;
    const Vec ev = vec_load_smem(ring + (size_t)slot * dim, dim, lane);
    __syncwarp();                        // every lane has its copy: the slot may be refilled
    if (lane == 0 && j + RING < n_loop) {
      ptx::fence_proxy_async();          // generic-proxy reads above, async-proxy write below
      request(j + RING);
    }
    const long long e = (long long)(code & ROW_MASK);
    FastNeg n;
    if (REL && (code & CODE_REL)) {      // warp-uniform
      fast_rel_negative<MODEL, LOSS>(pp, rl, ev, n);
      pair_forward<BWD, LOSS>(a, idx, lane, pp.pos, n.neg, loss);
      if constexpr (BWD)
        fast_rel_negative_backward<MODEL, LOSS>(pp, ev, n, a.margin, g, gr.rel0 + (size_t)e * dim, dim, lane, acc, rl);
      continue;
    }
    const bool head = (code & 0x80000000u) != 0u;   // warp-uniform
    fast_negative<MODEL, BWD>(pp, ab, ev, head, n);
    pair_forward<BWD, LOSS>(a, idx, lane, pp.pos, n.neg, loss);
    if constexpr (BWD)
      fast_negative_backward<MODEL, LOSS>(pp, ab, ev, head, n, a.margin, g, gr.ent0 + (size_t)e * dim, dim, lane, acc);
  }
  if constexpr (BWD)
    fast_positive_backward<MODEL, LOSS, REL>(pp, ab, acc, g,
                                             SHARD ? a.grad_hrows + (size_t)w * dim : gr.ent0 + (size_t)hi * dim,
                                             SHARD ? a.grad_trows + (size_t)w * dim : gr.ent0 + (size_t)ti * dim,
                                             gr.rel0 + (size_t)ri * dim, dim, lane, &rl);
  else if (lane == 0) atomicAdd(a.loss, loss);
}

template <int MODEL, bool BWD, int MINB = 0, bool SHARD = false, int LOSS = KGE_LOSS_MARGIN>
__global__ void __launch_bounds__(WARPS_PER_BLOCK * 32, MINB == 0 ? 1 : MINB)
margin_step_ring_kernel(MarginStepParams a, TrainGrads gr, const float* __restrict__ gloss) {
  ring_step<MODEL, BWD, SHARD, LOSS, false>(a, gr, gloss);
}

template <int MODEL, bool BWD, bool SHARD, int LOSS>
__global__ void __launch_bounds__(WARPS_PER_BLOCK * 32, 1)
margin_step_ring_rel_kernel(MarginStepParams a, TrainGrads gr, const float* __restrict__ gloss) {
  ring_step<MODEL, BWD, SHARD, LOSS, true>(a, gr, gloss);
}

template <int MODEL, bool BWD, bool SHARD, int LOSS>
__global__ void __launch_bounds__(WARPS_PER_BLOCK * 32, 1)
margin_step_ring_pos_kernel(MarginStepParams a, TrainGrads gr, const float* __restrict__ gloss, PosCSR pc) {
  ring_step<MODEL, BWD, SHARD, LOSS, false, true>(a, gr, gloss, pc);
}

__host__ inline size_t ring_smem_bytes(const MarginStepParams& a) {
  const size_t per_warp = (size_t)RING * a.dim * 4 + (size_t)((a.n_neg + 3) & ~3) * 4 + RING * sizeof(uint64_t);
  return WARPS_PER_BLOCK * ((per_warp + 127) & ~(size_t)127);
}
// KGE_TRAIN_RING=0 selects the register-resident form (margin_step_fast_kernel; the sharded step then
// takes the generic kernels).  Codes hold 31-bit row numbers: of the table, or of the shard; a relation
// step's codes (a.n_rel > 0) 30-bit row numbers of either table.
__host__ inline bool ring_step_ok(const MarginStepParams& a) {
  static const bool enabled = [] { const char* v = getenv("KGE_TRAIN_RING"); return !(v && v[0] == '0'); }();
  const long long rows = a.hrows ? a.n_rows : a.n_ent;
  const long long row_limit = a.n_rel > 0 ? 0x3FFFFFFFll : 0x7FFFFFFFll;
  return enabled && a.n_neg <= 8192 && rows < row_limit && a.n_rel < 0x3FFFFFFFll && ring_smem_bytes(a) <= 96 * 1024;
}

// REL: margin_step_ring_rel_kernel, POS: margin_step_ring_pos_kernel, which also takes the CSR (MINB is 0 there)
template <int MODEL, bool BWD, int MINB, bool SHARD, int LOSS, bool REL, bool POS>
constexpr auto ring_kernel() {
  if constexpr (POS) return margin_step_ring_pos_kernel<MODEL, BWD, SHARD, LOSS>;
  else if constexpr (REL) return margin_step_ring_rel_kernel<MODEL, BWD, SHARD, LOSS>;
  else return margin_step_ring_kernel<MODEL, BWD, MINB, SHARD, LOSS>;
}

template <int MODEL, bool BWD, int MINB, bool SHARD = false, int LOSS = KGE_LOSS_MARGIN, bool REL = false,
          bool POS = false>
cudaError_t launch_ring_variant(const MarginStepParams& a, const TrainGrads& gr, const float* gloss, cudaStream_t st,
                                const PosCSR& pc = PosCSR{}) {
  constexpr auto kernel = ring_kernel<MODEL, BWD, MINB, SHARD, LOSS, REL, POS>();
  const size_t smem = ring_smem_bytes(a);
  if (smem > 48 * 1024) {
    const cudaError_t e = set_attribute_once<kernel>(cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024);
    if (e != cudaSuccess) return e;
  }
  const unsigned blocks = (unsigned)((a.b + WARPS_PER_BLOCK - 1) / WARPS_PER_BLOCK);
  if constexpr (POS) kernel<<<blocks, WARPS_PER_BLOCK * 32, smem, st>>>(a, gr, gloss, pc);
  else kernel<<<blocks, WARPS_PER_BLOCK * 32, smem, st>>>(a, gr, gloss);
  return cudaGetLastError();
}

// One ring kernel per (entity, relation or positional step, loss kind, sharded).  KGE_TRAIN_BWD_BLOCKS=5 holds the
// backward kernel to 96 registers (5 CTAs = 20 warps per SM; the unsharded entity step with the margin
// loss only).
template <int MODEL, bool BWD>
cudaError_t launch_ring(const MarginStepParams& a, const TrainGrads& gr, const float* gloss, cudaStream_t st,
                        const PosCSR& pc) {
  auto by_shard = [&](auto loss) -> cudaError_t {
    constexpr int LOSS = decltype(loss)::value;
    if (pc.head_offs)
      return a.hrows ? launch_ring_variant<MODEL, BWD, 0, true, LOSS, false, true>(a, gr, gloss, st, pc)
                     : launch_ring_variant<MODEL, BWD, 0, false, LOSS, false, true>(a, gr, gloss, st, pc);
    if (a.n_rel > 0)
      return a.hrows ? launch_ring_variant<MODEL, BWD, 0, true, LOSS, true>(a, gr, gloss, st)
                     : launch_ring_variant<MODEL, BWD, 0, false, LOSS, true>(a, gr, gloss, st);
    if (a.hrows) return launch_ring_variant<MODEL, BWD, 0, true, LOSS>(a, gr, gloss, st);
    if constexpr (BWD && LOSS == KGE_LOSS_MARGIN) {
      static const bool tight = [] { const char* v = getenv("KGE_TRAIN_BWD_BLOCKS"); return v && v[0] == '5'; }();
      if (tight) return launch_ring_variant<MODEL, true, 5, false, LOSS>(a, gr, gloss, st);
    }
    return launch_ring_variant<MODEL, BWD, 0, false, LOSS>(a, gr, gloss, st);
  };
  switch (a.loss_kind) {
    case KGE_LOSS_LOGISTIC: return by_shard(std::integral_constant<int, KGE_LOSS_LOGISTIC>{});
    case KGE_LOSS_BCE: return by_shard(std::integral_constant<int, KGE_LOSS_BCE>{});
    default: return by_shard(std::integral_constant<int, KGE_LOSS_MARGIN>{});
  }
}

// margin_step_fast_kernel (the register-resident form, KGE_TRAIN_RING=0) has the margin loss only; the
// other losses take the generic kernels there
__host__ inline bool fast_step_ok(const MarginStepParams& a) {
  return (a.model == KGE_TRANSE_L1 || a.model == KGE_TRANSE_L2 || a.model == KGE_DISTMULT) &&
         a.dim % 4 == 0 && a.dim <= FAST_MAX_DIM;
}

// MarginLoss, LogisticLoss, BinaryCrossEntropyLoss (utils/losses.py:12-112), sum-reduced: pair_loss_term /
// pair_loss_grads element by element.  `margin` is read by the margin loss only.
__global__ void pair_loss_fwd_kernel(int kind, float margin, const float* __restrict__ pos,
                                     const float* __restrict__ neg, long long n, float* __restrict__ loss) {
  float s = 0.f;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (long long)gridDim.x * blockDim.x)
    s += pair_loss_term(kind, margin, pos[i], neg[i]);
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0 && s != 0.f) atomicAdd(loss, s);
}

__global__ void pair_loss_bwd_kernel(int kind, float margin, const float* __restrict__ pos,
                                     const float* __restrict__ neg, long long n, const float* __restrict__ gloss,
                                     float* __restrict__ gpos, float* __restrict__ gneg) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  pair_loss_grads(kind, margin, *gloss, pos[i], neg[i], gpos + i, gneg + i);
}

inline unsigned blocks_for_warps(long long warps) {
  return (unsigned)((warps + WARPS_PER_BLOCK - 1) / WARPS_PER_BLOCK);
}

// grad_plane[idx[i] - ent_lo] += rows[i][plane] for the ids this shard holds (the inverse of
// gather_rows_kernel); one warp per (i, plane) row, atomics because ids repeat.
__global__ void scatter_rows_add_kernel(float* __restrict__ grad0, float* __restrict__ grad1, int planes,
                                        long long ent_lo, long long n_rows, int dim,
                                        const int64_t* __restrict__ idx, long long n,
                                        const float* __restrict__ rows) {
  const long long w = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= n * planes) return;
  const long long i = w / planes;
  const int pl = (int)(w - i * planes);
  const long long row = idx[i] - ent_lo;
  if (row < 0 || row >= n_rows) return;
  const Planes<float> p = table_planes(grad0, grad1, planes, (size_t)row * dim);
  float* dst = pl == 0 ? p.p0 : (pl == 1 ? p.p1 : p.p2);
  const float* src = rows + (size_t)w * dim;
  for (int k = lane; k < dim; k += 32) atomicAdd(dst + k, src[k]);
}

}  // namespace

cudaError_t launch_scatter_rows_add(float* grad0, float* grad1, int planes, int64_t ent_lo, int64_t n_rows,
                                    int dim, const int64_t* idx, int64_t n, const float* rows, cudaStream_t st) {
  const long long warps = (long long)n * planes;
  if (warps <= 0) return cudaSuccess;
  scatter_rows_add_kernel<<<blocks_for_warps(warps), WARPS_PER_BLOCK * 32, 0, st>>>(grad0, grad1, planes, ent_lo,
                                                                                    n_rows, dim, idx, n, rows);
  return cudaGetLastError();
}

cudaError_t launch_score_triples_fwd(int model, int dim, const TrainTables& tb, const int64_t* h,
                                     const int64_t* t, const int64_t* r, int64_t n, float* out,
                                     cudaStream_t st) {
  if (n <= 0) return cudaSuccess;
  score_triples_fwd_kernel<<<blocks_for_warps(n), WARPS_PER_BLOCK * 32, 0, st>>>(model, dim, tb, h, t,
                                                                                 r, n, out);
  return cudaGetLastError();
}

cudaError_t launch_score_triples_bwd(int model, int dim, const TrainTables& tb, const TrainGrads& gr,
                                     const int64_t* h, const int64_t* t, const int64_t* r, int64_t n,
                                     const float* gout, cudaStream_t st) {
  if (n <= 0) return cudaSuccess;
  score_triples_bwd_kernel<<<blocks_for_warps(n), WARPS_PER_BLOCK * 32, 0, st>>>(model, dim, tb, gr, h,
                                                                                 t, r, n, gout);
  return cudaGetLastError();
}

cudaError_t launch_transh_score_fwd(const float* ent, const float* rel, const float* norm_vect, int dim,
                                    const int64_t* h, const int64_t* t, const int64_t* r, int64_t n, float* out,
                                    cudaStream_t st) {
  if (n <= 0) return cudaSuccess;
  transh_score_fwd_kernel<<<blocks_for_warps(n), WARPS_PER_BLOCK * 32, 0, st>>>(ent, rel, norm_vect, dim, h, t, r,
                                                                                n, out);
  return cudaGetLastError();
}

cudaError_t launch_transh_score_bwd(const float* ent, const float* rel, const float* norm_vect, float* g_ent,
                                    float* g_rel, float* g_norm_vect, int dim, const int64_t* h, const int64_t* t,
                                    const int64_t* r, int64_t n, const float* gout, cudaStream_t st) {
  if (n <= 0) return cudaSuccess;
  transh_score_bwd_kernel<<<blocks_for_warps(n), WARPS_PER_BLOCK * 32, 0, st>>>(
      ent, rel, norm_vect, g_ent, g_rel, g_norm_vect, dim, h, t, r, n, gout);
  return cudaGetLastError();
}

cudaError_t launch_transd_score_fwd(const float* ent, const float* rel, const float* ent_proj,
                                    const float* rel_proj, int ent_dim, int rel_dim, const int64_t* h,
                                    const int64_t* t, const int64_t* r, int64_t n, float* out, cudaStream_t st) {
  if (n <= 0) return cudaSuccess;
  transd_score_fwd_kernel<<<blocks_for_warps(n), WARPS_PER_BLOCK * 32, 0, st>>>(ent, rel, ent_proj, rel_proj, ent_dim,
                                                                                rel_dim, h, t, r, n, out);
  return cudaGetLastError();
}

cudaError_t launch_transd_score_bwd(const float* ent, const float* rel, const float* ent_proj,
                                    const float* rel_proj, float* g_ent, float* g_rel, float* g_ent_proj,
                                    float* g_rel_proj, int ent_dim, int rel_dim, const int64_t* h, const int64_t* t,
                                    const int64_t* r, int64_t n, const float* gout, cudaStream_t st) {
  if (n <= 0) return cudaSuccess;
  transd_score_bwd_kernel<<<blocks_for_warps(n), WARPS_PER_BLOCK * 32, 0, st>>>(
      ent, rel, ent_proj, rel_proj, g_ent, g_rel, g_ent_proj, g_rel_proj, ent_dim, rel_dim, h, t, r, n, gout);
  return cudaGetLastError();
}

cudaError_t launch_corrupt_batch(const int64_t* h, const int64_t* t, const int64_t* r, int64_t b,
                                 int n_neg, const float* probs, int64_t n_ent, uint64_t seed,
                                 uint64_t offset, int64_t* nh, int64_t* nt, cudaStream_t st) {
  const long long n = (long long)b * n_neg;
  if (n <= 0) return cudaSuccess;
  corrupt_batch_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(h, t, r, b, n_neg, probs, n_ent,
                                                                     seed, offset, nh, nt);
  return cudaGetLastError();
}

cudaError_t launch_corrupt_batch_rel(const int64_t* h, const int64_t* t, const int64_t* r, int64_t b,
                                     int n_neg, const float* probs, int64_t n_ent, int64_t n_rel, float rel_share,
                                     uint64_t seed, uint64_t offset, int64_t* nh, int64_t* nt, int64_t* nr,
                                     cudaStream_t st) {
  const long long n = (long long)b * n_neg;
  if (n <= 0) return cudaSuccess;
  corrupt_batch_rel_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(h, t, r, b, n_neg, probs, n_ent, n_rel,
                                                                         rel_share, seed, offset, nh, nt, nr);
  return cudaGetLastError();
}

namespace {
// f(std::integral_constant<int, MODEL>{}) for the models of the ring and register-resident forms
// (fast_step_ok)
template <class F>
cudaError_t with_fast_model(int model, F&& f) {
  switch (model) {
    case KGE_TRANSE_L1: return f(std::integral_constant<int, KGE_TRANSE_L1>{});
    case KGE_TRANSE_L2: return f(std::integral_constant<int, KGE_TRANSE_L2>{});
    default: return f(std::integral_constant<int, KGE_DISTMULT>{});
  }
}

// The ring kernel where it applies; else, for an unsharded entity step with the margin loss, the
// register-resident form; else the generic kernels.  An entity-sharded step (a.hrows) that holds no
// rows scores no negative.
//
// A relation-corrupting step (a.n_rel > 0): at rel_share >= 1 its draws are the entity step's
// (draw_rel), so without caller negatives or an nr_out to fill it is that step.  Otherwise TransE-L1 /
// L2 and DistMult take the ring kernel's relation kind (margin_step_ring_rel_kernel) where the ring
// applies; everything else, and KGE_TRAIN_RING=0, takes the generic kernels, which score a negative from
// its own (nh, nt, nr).
//
// A positional step (pc.head_offs set, n_rel 0): the ring kernel's positional kind
// (margin_step_ring_pos_kernel) where the ring applies, else the generic kernels -- never the register-resident
// form, as for the relation step.
template <bool BWD>
cudaError_t launch_margin_step(MarginStepParams a, const TrainGrads& gr, const float* gloss, cudaStream_t st,
                               const PosCSR& pc) {
  if (a.n_rel > 0 && a.rel_share >= 1.f && !a.nh && !a.nr_out) a.n_rel = 0;
  const bool shard = a.hrows != nullptr;
  if (a.b <= 0 || (shard && a.n_rows <= 0)) return cudaSuccess;
  const unsigned blocks = blocks_for_warps(a.b);
  if (fast_step_ok(a) && ring_step_ok(a))
    return with_fast_model(a.model, [&](auto m) { return launch_ring<decltype(m)::value, BWD>(a, gr, gloss, st, pc); });
  if (a.n_rel <= 0 && !pc.head_offs) {   // the register-resident form has no relation or positional kind
    if (!shard && fast_step_ok(a) && a.loss_kind == KGE_LOSS_MARGIN) {
      return with_fast_model(a.model, [&](auto m) {
        margin_step_fast_kernel<decltype(m)::value, BWD><<<blocks, WARPS_PER_BLOCK * 32, 0, st>>>(a, gr, gloss);
        return cudaGetLastError();
      });
    }
  }
  if constexpr (BWD) {
    if (shard) margin_step_shard_bwd_kernel<<<blocks, WARPS_PER_BLOCK * 32, 0, st>>>(a, gr, gloss, pc);
    else margin_step_bwd_kernel<<<blocks, WARPS_PER_BLOCK * 32, 0, st>>>(a, gr, gloss, pc);
  } else {
    if (shard) margin_step_shard_fwd_kernel<<<blocks, WARPS_PER_BLOCK * 32, 0, st>>>(a, pc);
    else margin_step_fwd_kernel<<<blocks, WARPS_PER_BLOCK * 32, 0, st>>>(a, pc);
  }
  return cudaGetLastError();
}
}  // namespace

cudaError_t launch_margin_step_fwd(const MarginStepParams& a, cudaStream_t st, const PosCSR& pos) {
  return launch_margin_step<false>(a, TrainGrads{nullptr, nullptr, nullptr, nullptr}, nullptr, st, pos);
}

cudaError_t launch_margin_step_bwd(const MarginStepParams& a, const TrainGrads& gr, const float* gloss,
                                   cudaStream_t st, const PosCSR& pos) {
  return launch_margin_step<true>(a, gr, gloss, st, pos);
}

cudaError_t launch_pair_loss_fwd(int kind, float margin, const float* pos, const float* neg, int64_t n,
                                 float* loss, cudaStream_t st) {
  if (n <= 0) return cudaSuccess;
  const unsigned blocks = (unsigned)((n + 255) / 256 < 1184 ? (n + 255) / 256 : 1184);
  pair_loss_fwd_kernel<<<blocks, 256, 0, st>>>(kind, margin, pos, neg, n, loss);
  return cudaGetLastError();
}

cudaError_t launch_pair_loss_bwd(int kind, float margin, const float* pos, const float* neg, int64_t n,
                                 const float* gloss, float* gpos, float* gneg, cudaStream_t st) {
  if (n <= 0) return cudaSuccess;
  pair_loss_bwd_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(kind, margin, pos, neg, n, gloss, gpos, gneg);
  return cudaGetLastError();
}

}  // namespace kge
