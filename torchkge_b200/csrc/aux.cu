// Everything around the dense scan: table packing, query-row gather, query preparation,
// the sparse pair scorer (true scores, filter sets) and rank finalisation.  These kernels
// move little data compared with the scan; they are written for coalescing and exactness,
// not tuned further.
#include "kernels.h"

namespace kge {

int elem_kind_for(int model, int side) {
  const bool tail = side == KGE_SIDE_TAIL;
  if (side == KGE_SIDE_REL) {
    // candidates are relation rows, the query is the (h, t) pair:
    //   TransE   -diss(h + c, t)                       interfaces.py:261-272  ((c + h) - t: fp add commutes)
    //   DistMult ((h * c) * t).sum                     bilinear.py:241-245
    //   ComplEx  ((re_h re_t + im_h im_t) re_c + (re_h im_t - im_h re_t) im_c).sum   bilinear.py:524-528
    switch (model) {
      case KGE_TRANSE_L1: return EL_L1_HEAD;
      case KGE_TRANSE_L2: return EL_L2_HEAD;
      case KGE_DISTMULT: return EL_DOT_MID;
      case KGE_COMPLEX: return EL_DOT2;
      //   Analogy  (sc_c (sc_h sc_t) + re_c (re_h re_t + im_h im_t) + im_c (re_h im_t - im_h re_t)).sum   bilinear.py:709-712
      case KGE_ANALOGY: return EL_DOT3;
      default: return -1;  // RESCAL (batched matmul in the reference) and RotatE: not on this path
    }
  }
  if (side != KGE_SIDE_TAIL && side != KGE_SIDE_HEAD) return -1;
  switch (model) {
    case KGE_TRANSE_L1: return tail ? EL_L1_TAIL : EL_L1_HEAD;
    case KGE_TRANSE_L2: return tail ? EL_L2_TAIL : EL_L2_HEAD;
    case KGE_DISTMULT:
    case KGE_RESCAL: return EL_DOT1;
    case KGE_COMPLEX: return EL_DOT2;
    case KGE_ROTATE: return EL_ROT;
    case KGE_TORUSE_L1: return tail ? EL_TL1_TAIL : EL_TL1_HEAD;
    case KGE_TORUSE_L2: return tail ? EL_TL2_TAIL : EL_TL2_HEAD;
    case KGE_ANALOGY: return EL_DOT3;
    default: return -1;
  }
}

int elem_qw(int el) {
  switch (el) {
    case EL_DOT1: case EL_L1_TAIL: case EL_L2_TAIL: case EL_TL1_TAIL: case EL_TL2_TAIL: return 1;
    case EL_DOT3: return 3;
    default: return 2;
  }
}

int elem_cw(int el) { return el == EL_DOT3 ? 3 : ((el == EL_DOT2 || el == EL_ROT) ? 2 : 1); }

namespace {

// ------------------------------------------------------------------------------------
// pack_table: grid (n_ct, ceil(dim/32)); block 256.  Reads a [TILE_C rows][32 k] patch with
// coalesced 128-B row segments, transposes it through shared memory and writes, for each of
// the 32 embedding indices, one 512-B candidate-major row at its schedule position.
// ------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) pack_table_kernel(const float* __restrict__ ent0,
                                                         const float* __restrict__ ent1,
                                                         int planes, long long n_rows, int dim,
                                                         const int32_t* __restrict__ inv_perm,
                                                         float* __restrict__ packed) {
  __shared__ float tile[32][TILE_C + 1];
  const long long ct = blockIdx.x;
  const int k0 = blockIdx.y * 32;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int pl = 0; pl < planes; ++pl) {
    const float* ent = pl == 0 ? ent0 : (pl == 1 ? ent1 : third_plane(ent0, ent1));
    for (int r = warp; r < TILE_C; r += 8) {
      const long long row = ct * TILE_C + r;
      const int k = k0 + lane;
      float v = 0.f;
      if (row < n_rows && k < dim) v = ent[(size_t)row * dim + k];
      tile[lane][r] = v;
    }
    __syncthreads();
    for (int kk = warp; kk < 32; kk += 8) {
      const int k = k0 + kk;
      if (k < dim) {
        const int pos = inv_perm[k];
        float* dst = packed + (((size_t)ct * dim + pos) * planes + pl) * TILE_C;
        for (int c = lane; c < TILE_C; c += 32) dst[c] = tile[kk][c];
      }
    }
    __syncthreads();
  }
}

// out[i][plane][dim] = ent_plane[idx[i]-ent_lo] or 0.  One warp per (i, plane) row.
__global__ void gather_rows_kernel(const float* __restrict__ ent0, const float* __restrict__ ent1,
                                   int planes, long long ent_lo, long long n_rows, int dim,
                                   const int64_t* __restrict__ idx, long long n,
                                   float* __restrict__ out) {
  const long long w = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= n * planes) return;
  const long long i = w / planes;
  const int pl = (int)(w - i * planes);
  const long long row = idx[i] - ent_lo;
  const float* ent = pl == 0 ? ent0 : (pl == 1 ? ent1 : third_plane(ent0, ent1));
  float* dst = out + (size_t)w * dim;
  const bool own = row >= 0 && row < n_rows;
  for (int k = lane; k < dim; k += 32) dst[k] = own ? ent[(size_t)row * dim + k] : 0.f;
}

// Query preparation for the element-wise models: the (b, d) tensor algebra that precedes the
// broadcast against all candidates, with the reference's operation order.
//   TransE tail  q0 = h + r                                    interfaces.py:253
//   TransE head  q0 = r, q1 = t                                interfaces.py:258-259
//   DistMult     tail q0 = h*r ; head q0 = r*t                 bilinear.py:234, 239
//   ComplEx tail q0 = re_h*re_r - im_h*im_r ; q1 = re_h*im_r + im_h*re_r   bilinear.py:514-515
//   ComplEx head q0 = re_r*re_t + im_r*im_t ; q1 = re_r*im_t - im_r*re_t   bilinear.py:521-522
//   RotatE       same algebra as ComplEx with (rel0, rel1) = (cos, sin) of the phases:
//                tail q = h o r ; head q = t o conj(r)
//   Analogy      DistMult on the scalar plane, ComplEx on the (real, imaginary) planes  bilinear.py:694-706
// Relation prediction (side = KGE_SIDE_REL, candidates = relation rows; rel0/rel1 unused):
//   TransE / DistMult  q0 = h, q1 = t
//   ComplEx  q0 = re_h*re_t + im_h*im_t ; q1 = re_h*im_t - im_h*re_t       bilinear.py:527-528
__global__ void prep_queries_kernel(int model, int side, int dim, long long n,
                                    const float* __restrict__ hrows,
                                    const float* __restrict__ trows,
                                    const float* __restrict__ rel0,
                                    const float* __restrict__ rel1,
                                    const int64_t* __restrict__ r_idx,
                                    float* __restrict__ qplain) {
  const long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (gid >= n * dim) return;
  const long long i = gid / dim;
  const int k = (int)(gid - i * dim);
  const bool tail = side == KGE_SIDE_TAIL;
  if (side == KGE_SIDE_REL) {
    if (model == KGE_ANALOGY) {   // bilinear.py:709-712; planes (scalar, real, imaginary)
      const float* hp = hrows + (size_t)i * 3 * dim + k;
      const float* tp = trows + (size_t)i * 3 * dim + k;
      const float sc_h = hp[0], re_h = hp[dim], im_h = hp[2 * dim];
      const float sc_t = tp[0], re_t = tp[dim], im_t = tp[2 * dim];
      float* q = qplain + (size_t)i * 3 * dim + k;
      q[0] = __fmul_rn(sc_h, sc_t);
      q[dim] = __fadd_rn(__fmul_rn(re_h, re_t), __fmul_rn(im_h, im_t));
      q[2 * dim] = __fsub_rn(__fmul_rn(re_h, im_t), __fmul_rn(im_h, re_t));
    } else if (model == KGE_COMPLEX) {
      const float re_h = hrows[((size_t)i * 2 + 0) * dim + k], im_h = hrows[((size_t)i * 2 + 1) * dim + k];
      const float re_t = trows[((size_t)i * 2 + 0) * dim + k], im_t = trows[((size_t)i * 2 + 1) * dim + k];
      qplain[((size_t)i * 2 + 0) * dim + k] = __fadd_rn(__fmul_rn(re_h, re_t), __fmul_rn(im_h, im_t));
      qplain[((size_t)i * 2 + 1) * dim + k] = __fsub_rn(__fmul_rn(re_h, im_t), __fmul_rn(im_h, re_t));
    } else {
      qplain[((size_t)i * 2 + 0) * dim + k] = hrows[(size_t)i * dim + k];
      qplain[((size_t)i * 2 + 1) * dim + k] = trows[(size_t)i * dim + k];
    }
    return;
  }
  const long long r = r_idx ? r_idx[i] : i;  // null r_idx: rel tables hold one row per query
  switch (model) {
    case KGE_TRANSE_L1:
    case KGE_TRANSE_L2:
    case KGE_TORUSE_L1:
    case KGE_TORUSE_L2: {
      const float rv = rel0[(size_t)r * dim + k];
      if (tail) {
        qplain[(size_t)i * dim + k] = __fadd_rn(hrows[(size_t)i * dim + k], rv);
      } else {
        qplain[((size_t)i * 2 + 0) * dim + k] = rv;
        qplain[((size_t)i * 2 + 1) * dim + k] = trows[(size_t)i * dim + k];
      }
      break;
    }
    case KGE_DISTMULT: {
      const float rv = rel0[(size_t)r * dim + k];
      const float ev = tail ? hrows[(size_t)i * dim + k] : trows[(size_t)i * dim + k];
      qplain[(size_t)i * dim + k] = tail ? __fmul_rn(ev, rv) : __fmul_rn(rv, ev);
      break;
    }
    case KGE_COMPLEX:
    case KGE_ROTATE: {
      const float re_r = rel0[(size_t)r * dim + k];
      const float im_r = rel1[(size_t)r * dim + k];
      float q0, q1;
      if (tail) {
        const float re_h = hrows[((size_t)i * 2 + 0) * dim + k];
        const float im_h = hrows[((size_t)i * 2 + 1) * dim + k];
        q0 = __fsub_rn(__fmul_rn(re_h, re_r), __fmul_rn(im_h, im_r));
        q1 = __fadd_rn(__fmul_rn(re_h, im_r), __fmul_rn(im_h, re_r));
      } else {
        const float re_t = trows[((size_t)i * 2 + 0) * dim + k];
        const float im_t = trows[((size_t)i * 2 + 1) * dim + k];
        q0 = __fadd_rn(__fmul_rn(re_r, re_t), __fmul_rn(im_r, im_t));
        q1 = __fsub_rn(__fmul_rn(re_r, im_t), __fmul_rn(im_r, re_t));
      }
      qplain[((size_t)i * 2 + 0) * dim + k] = q0;
      qplain[((size_t)i * 2 + 1) * dim + k] = q1;
      break;
    }
    case KGE_ANALOGY: {
      // tail (bilinear.py:695-699): q = (sc_h sc_r, re_h re_r - im_h im_r, re_h im_r + im_h re_r)
      // head (bilinear.py:702-706): q = (sc_r sc_t, re_r re_t + im_r im_t, re_r im_t - im_r re_t)
      const float sc_r = rel0[(size_t)r * dim + k];
      const float re_r = rel1[(size_t)r * dim + k];
      const float im_r = third_plane(rel0, rel1)[(size_t)r * dim + k];
      const float* ep = (tail ? hrows : trows) + (size_t)i * 3 * dim + k;
      const float sc_e = ep[0], re_e = ep[dim], im_e = ep[2 * dim];
      float* q = qplain + (size_t)i * 3 * dim + k;
      if (tail) {
        q[0] = __fmul_rn(sc_e, sc_r);
        q[dim] = __fsub_rn(__fmul_rn(re_e, re_r), __fmul_rn(im_e, im_r));
        q[2 * dim] = __fadd_rn(__fmul_rn(re_e, im_r), __fmul_rn(im_e, re_r));
      } else {
        q[0] = __fmul_rn(sc_r, sc_e);
        q[dim] = __fadd_rn(__fmul_rn(re_r, re_e), __fmul_rn(im_r, im_e));
        q[2 * dim] = __fsub_rn(__fmul_rn(re_r, im_e), __fmul_rn(im_r, re_e));
      }
      break;
    }
    default: break;
  }
}

// RESCAL query preparation: tail q = h^T M_r (bilinear.py:113), head q = M_r t
// (bilinear.py:108); M_r = rel_mat[r] viewed (dim, dim) row-major.  One thread per output
// component, in the reference's (oneMKL / ATen) summation order: reduce.cuh,
// rescal_query_component.  Consecutive threads own consecutive components: the tail side reads
// M[k][j..] coalesced, the head side walks its own row (L1-resident, tiny next to the scan).
__global__ void prep_rescal_kernel(int side, int dim, long long n,
                                   const float* __restrict__ hrows,
                                   const float* __restrict__ trows,
                                   const float* __restrict__ rel_mat,
                                   const int64_t* __restrict__ r_idx,
                                   float* __restrict__ qplain) {
  const long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (gid >= n * dim) return;
  const long long i = gid / dim;
  const int j = (int)(gid - i * dim);
  const float* M = rel_mat + (size_t)(r_idx ? r_idx[i] : i) * dim * dim;
  const bool tail = side == KGE_SIDE_TAIL;
  const float* vec = (tail ? hrows : trows) + (size_t)i * dim;
  qplain[(size_t)i * dim + j] = rescal_query_component(tail, dim, j, vec, M);
}

// qpacked[qt][pos][plane][TILE_Q]; thread per output float, zero padded past n.
__global__ void pack_queries_kernel(const float* __restrict__ qplain, int qw, int dim,
                                    long long n, long long n_qt,
                                    const int32_t* __restrict__ perm,
                                    float* __restrict__ qpacked) {
  const long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long total = n_qt * dim * qw * TILE_Q;
  if (gid >= total) return;
  const int ql = (int)(gid % TILE_Q);
  long long rest = gid / TILE_Q;
  const int pl = (int)(rest % qw);
  rest /= qw;
  const int pos = (int)(rest % dim);
  const long long qt = rest / dim;
  const long long i = qt * TILE_Q + ql;
  float v = 0.f;
  if (i < n) v = qplain[((size_t)i * qw + pl) * dim + perm[pos]];
  qpacked[gid] = v;
}

__global__ void fill_f32_kernel(float* dst, float value, long long n) {
  const long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (gid < n) dst[gid] = value;
}

// One (query, candidate-row) score by replaying the schedule: same device functions as the
// dense scan, hence bit-identical results.
template <int EL, bool CASC>
__device__ __forceinline__ float pair_score(int dim, const float* __restrict__ q0p,
                                            const float* __restrict__ q1p,
                                            const float* __restrict__ c0p,
                                            const float* __restrict__ c1p,
                                            const int32_t* __restrict__ perm,
                                            const uint8_t* __restrict__ code) {
  Acc r;
  acc_reset(r);
  for (int pos = 0; pos < dim; ++pos) {
    const int k = perm[pos];
    acc_step<EL, CASC>(r, code[pos], q0p[k], q1p[k], c0p[k], c1p[k]);
  }
  return acc_finish<EL>(r);
}

// s_true[i] = score(query i, its true row).  Chain-parallel like the filter pass: 8 lanes per query for
// the L2 norm, 32 for the cascade sum (pair_score_chains: same bits as the schedule replay), one lane
// for the sequential L1 norm and for dims below 8.
template <int EL, bool CASC>
__global__ void true_scores_kernel(int dim, long long n, const float* __restrict__ qplain,
                                   const float* __restrict__ rows,
                                   const int32_t* __restrict__ perm,
                                   const uint8_t* __restrict__ code, float* __restrict__ s_true) {
  constexpr int QW = ElemTraits<EL>::QW, CW = ElemTraits<EL>::CW;
  constexpr int RED = ElemTraits<EL>::RED;
  constexpr int LANES = RED == RED_SEQ ? 1 : (RED == RED_NORM2 ? 8 : 32);
  constexpr int PER_WARP = 32 / LANES;
  const int lane = threadIdx.x & 31;
  const long long warp_global = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long base = warp_global * PER_WARP;
  if (base >= n) return;
  const long long i = base + lane / LANES;
  const bool valid = i < n;
  const long long ii = valid ? i : base;     // idle groups redo the first query (shuffles stay uniform)
  const float* q0 = qplain + (size_t)ii * QW * dim;
  const float* q1 = q0 + (size_t)(QW - 1) * dim;
  const float* c0 = rows + (size_t)ii * CW * dim;
  const float* c1 = c0 + (size_t)(CW - 1) * dim;
  const float* qm = q0 + (size_t)(QW / 2) * dim;   // middle plane (three-plane kinds)
  const float* cm = c0 + (size_t)(CW / 2) * dim;
  float s;
  if constexpr (RED == RED_SEQ) {
    s = pair_score<EL, CASC>(dim, q0, q1, c0, c1, perm, code);
  } else {
    if (RED == RED_SUM && dim < 8) s = pair_score_natural<EL>(dim, q0, q1, c0, c1, qm, cm);
    else s = pair_score_chains<EL>(dim, q0, q1, c0, c1, lane, qm, cm);
  }
  if (valid && (lane % LANES) == 0) s_true[i] = s;
}

// Filter pass.  For every CSR entry c of query i held by this shard:
//   filt_sub[i] += [s(i,c) >= s_true(i)] - [s_true(i) == -inf]
// (filter_scores writes -inf over the entry, modeling.py:100; get_rank then counts
// (-inf >= s_true) instead of (s >= s_true), operations.py:61).  Chain-parallel scoring: 8 lanes
// per entry for the L2 norm, 32 for the cascade sum (pair_score_chains), one lane for the
// sequential L1 norm (schedule replay).
template <int EL, bool CASC>
__global__ void filter_kernel(int dim, long long n, long long n_filt,
                              const float* __restrict__ qplain, const float* __restrict__ ent0,
                              const float* __restrict__ ent1, long long ent_lo,
                              long long n_rows, const int64_t* __restrict__ offs,
                              const int64_t* __restrict__ ids, const int32_t* __restrict__ qid,
                              const int32_t* __restrict__ perm,
                              const uint8_t* __restrict__ code, const float* __restrict__ s_true,
                              int32_t* __restrict__ filt_sub) {
  constexpr int QW = ElemTraits<EL>::QW, CW = ElemTraits<EL>::CW;
  constexpr int RED = ElemTraits<EL>::RED;
  constexpr int LANES = RED == RED_SEQ ? 1 : (RED == RED_NORM2 ? 8 : 32);  // lanes per entry
  constexpr int PER_WARP = 32 / LANES;
  const int lane = threadIdx.x & 31;
  const long long warp_global = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long n_warps = ((long long)gridDim.x * blockDim.x) >> 5;
  const bool small_sum = RED == RED_SUM && dim < 8;  // one-lane cascade: lane 0 scores alone
  for (long long base = warp_global * PER_WARP; base < n_filt; base += n_warps * PER_WARP) {
    const long long e = base + lane / LANES;
    const bool in_range = e < n_filt;
    const long long ee = in_range ? e : base;
    const long long row = ids[ee] - ent_lo;
    const bool held = in_range && row >= 0 && row < n_rows;
    const long long rr = held ? row : 0;
    // query owning CSR entry ee: given, or the largest i with offs[i] <= ee
    long long lo = 0, hi = n;
    if (qid != nullptr) {
      lo = qid[ee];
    } else {
      while (hi - lo > 1) {
        const long long mid = (lo + hi) >> 1;
        if (offs[mid] <= ee) lo = mid; else hi = mid;
      }
    }
    const long long i = lo;
    const float* q0 = qplain + (size_t)i * QW * dim;
    const float* q1 = q0 + (size_t)(QW - 1) * dim;
    const float* c0 = ent0 + (size_t)rr * dim;
    const float* c1 = (CW == 3 ? third_plane(ent0, ent1) : (CW == 2 ? ent1 : ent0)) + (size_t)rr * dim;
    const float* qm = q0 + (size_t)(QW / 2) * dim;   // middle plane (three-plane kinds)
    const float* cm = (CW == 3 ? ent1 : ent0) + (size_t)rr * dim;
    float s;
    if constexpr (RED == RED_SEQ) {
      s = pair_score<EL, CASC>(dim, q0, q1, c0, c1, perm, code);
    } else {
      if (small_sum) s = pair_score_natural<EL>(dim, q0, q1, c0, c1, qm, cm);
      else s = pair_score_chains<EL>(dim, q0, q1, c0, c1, lane, qm, cm);
    }
    const bool leader = (lane % LANES) == 0;
    if (held && leader) {
      const float st = s_true[i];
      const int v = (s >= st ? 1 : 0) - (st == -INFINITY ? 1 : 0);
      if (v != 0) atomicAdd(&filt_sub[i], v);
    }
  }
}

__global__ void finalize_kernel(const int32_t* __restrict__ raw, const int32_t* __restrict__ sub,
                                long long n, int64_t* __restrict__ ranks,
                                int64_t* __restrict__ filt_ranks) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int64_t r = raw[i];
  ranks[i] = r;
  filt_ranks[i] = r - (int64_t)sub[i];
}

// TransH: out[row] = projection of ent[row] on the hyperplane of normal w (reduce.cuh:
// transh_project_elem).  One warp per row; the lanes share the row's normal component nc.
__global__ void __launch_bounds__(256) transh_project_kernel(const float* __restrict__ ent,
                                                             const float* __restrict__ w, long long n_rows,
                                                             int dim, float* __restrict__ out) {
  const long long row = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= n_rows) return;   // whole warps leave together: the shuffles below see full warps
  const float* e = ent + (size_t)row * dim;
  const float nc = dim < 8 ? pair_score_natural<EL_DOT1>(dim, e, e, w, w)
                           : pair_score_chains<EL_DOT1>(dim, e, e, w, w, lane);
  float* o = out + (size_t)row * dim;
  for (int k = lane; k < dim; k += 32) o[k] = transh_project_elem(e[k], nc, w[k]);
}

// TransD: s[row] = (ent_proj[row] * ent[row]).sum() in ATen's order (reduce.cuh: transd_project_elem).
// One warp per row.
__global__ void __launch_bounds__(256) transd_scalars_kernel(const float* __restrict__ ent,
                                                             const float* __restrict__ ent_proj, long long n_rows,
                                                             int dim, float* __restrict__ s) {
  const long long row = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= n_rows) return;   // whole warps leave together: the shuffles below see full warps
  const float* e = ent + (size_t)row * dim;
  const float* p = ent_proj + (size_t)row * dim;
  const float v = dim < 8 ? pair_score_natural<EL_DOT1>(dim, p, p, e, e)
                          : pair_score_chains<EL_DOT1>(dim, p, p, e, e, lane);
  if (lane == 0) s[row] = v;
}

// TransD: out[row][j] = transd_project_elem(ent[row][j], s[row], rp[j]) for j < rel_dim, the entity rows
// read with their own stride ent_dim.  Element-wise: one thread per output element.
__global__ void __launch_bounds__(256) transd_project_kernel(const float* __restrict__ ent, int ent_dim,
                                                             const float* __restrict__ s,
                                                             const float* __restrict__ rp, long long total,
                                                             int rel_dim, float* __restrict__ out) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long x = (long long)blockIdx.x * blockDim.x + threadIdx.x; x < total; x += stride) {
    const long long row = x / rel_dim;
    const int j = (int)(x - row * rel_dim);
    out[x] = transd_project_elem(ent[(size_t)row * ent_dim + j], s[row], rp[j]);
  }
}

inline unsigned filter_blocks(long long n_filt) {
  const long long want = (n_filt + 3) / 4;  // >= one warp per entry group; grid-stride beyond
  return (unsigned)(want < 1 ? 1 : (want > 132LL * 64 ? 132LL * 64 : want));   // 64 blocks per H100 SM
}

inline unsigned blocks_for(long long n, int threads) {
  return (unsigned)((n + threads - 1) / threads);
}

}  // namespace

cudaError_t launch_pack_table(const float* ent0, const float* ent1, int planes, int64_t n_rows,
                              int dim, const int32_t* inv_perm, float* packed,
                              cudaStream_t stream) {
  if (n_rows <= 0) return cudaSuccess;
  const long long n_ct = (n_rows + TILE_C - 1) / TILE_C;
  dim3 grid((unsigned)n_ct, (unsigned)((dim + 31) / 32));
  pack_table_kernel<<<grid, 256, 0, stream>>>(ent0, ent1, planes, n_rows, dim, inv_perm, packed);
  return cudaGetLastError();
}

cudaError_t launch_gather_rows(const float* ent0, const float* ent1, int planes, int64_t ent_lo,
                               int64_t n_rows, int dim, const int64_t* idx, int64_t n,
                               float* out, cudaStream_t stream) {
  if (n <= 0) return cudaSuccess;
  const long long warps = (long long)n * planes;
  gather_rows_kernel<<<blocks_for(warps * 32, 256), 256, 0, stream>>>(
      ent0, ent1, planes, ent_lo, n_rows, dim, idx, n, out);
  return cudaGetLastError();
}

cudaError_t launch_prep_queries(int model, int side, int dim, int64_t n, const float* hrows,
                                const float* trows, const float* rel0, const float* rel1,
                                const int64_t* r_idx, float* qplain, cudaStream_t stream) {
  if (n <= 0) return cudaSuccess;
  const long long total = (long long)n * dim;
  if (model == KGE_RESCAL)
    prep_rescal_kernel<<<blocks_for(total, 256), 256, 0, stream>>>(side, dim, n, hrows, trows,
                                                                   rel0, r_idx, qplain);
  else
    prep_queries_kernel<<<blocks_for(total, 256), 256, 0, stream>>>(
        model, side, dim, n, hrows, trows, rel0, rel1, r_idx, qplain);
  return cudaGetLastError();
}

cudaError_t launch_pack_queries(const float* qplain, int qw, int dim, int64_t n,
                                const int32_t* perm, float* qpacked, cudaStream_t stream) {
  if (n <= 0) return cudaSuccess;
  const long long n_qt = (n + TILE_Q - 1) / TILE_Q;
  const long long total = n_qt * dim * qw * TILE_Q;
  pack_queries_kernel<<<blocks_for(total, 256), 256, 0, stream>>>(qplain, qw, dim, n, n_qt, perm,
                                                                  qpacked);
  return cudaGetLastError();
}

cudaError_t launch_fill_f32(float* dst, float value, int64_t n, cudaStream_t stream) {
  if (n <= 0) return cudaSuccess;
  fill_f32_kernel<<<blocks_for(n, 256), 256, 0, stream>>>(dst, value, n);
  return cudaGetLastError();
}

cudaError_t launch_true_scores(int el, bool cascade, int dim, int64_t n, const float* qplain,
                               const float* rows, const int32_t* perm, const uint8_t* code,
                               float* s_true, cudaStream_t stream) {
  if (n <= 0) return cudaSuccess;
  return dispatch_elem(el, cascade, [&](auto kind, auto casc) {
    constexpr int EL = decltype(kind)::value;
    constexpr int LANES = ElemTraits<EL>::RED == RED_SEQ ? 1 : (ElemTraits<EL>::RED == RED_NORM2 ? 8 : 32);
    true_scores_kernel<EL, decltype(casc)::value><<<blocks_for(n * LANES, 128), 128, 0, stream>>>(
        dim, n, qplain, rows, perm, code, s_true);
    return cudaGetLastError();
  });
}

cudaError_t launch_filter(int el, bool cascade, int dim, int64_t n, int64_t n_filt,
                          const float* qplain, const float* ent0, const float* ent1,
                          int64_t ent_lo, int64_t n_rows, const int64_t* offs,
                          const int64_t* ids, const int32_t* qid, const int32_t* perm, const uint8_t* code,
                          const float* s_true, int32_t* filt_sub, cudaStream_t stream) {
  if (n <= 0 || n_filt <= 0) return cudaSuccess;
  return dispatch_elem(el, cascade, [&](auto kind, auto casc) {
    filter_kernel<decltype(kind)::value, decltype(casc)::value><<<filter_blocks(n_filt), 128, 0, stream>>>(
        dim, n, n_filt, qplain, ent0, ent1, ent_lo, n_rows, offs, ids, qid, perm, code, s_true, filt_sub);
    return cudaGetLastError();
  });
}

cudaError_t launch_transh_project(const float* ent, const float* w, int64_t n_rows, int dim, float* out,
                                  cudaStream_t stream) {
  if (n_rows <= 0) return cudaSuccess;
  transh_project_kernel<<<blocks_for(n_rows * 32, 256), 256, 0, stream>>>(ent, w, n_rows, dim, out);
  return cudaGetLastError();
}

cudaError_t launch_transd_entity_scalars(const float* ent, const float* ent_proj, int64_t n_rows, int ent_dim,
                                         float* s, cudaStream_t stream) {
  if (n_rows <= 0) return cudaSuccess;
  transd_scalars_kernel<<<blocks_for(n_rows * 32, 256), 256, 0, stream>>>(ent, ent_proj, n_rows, ent_dim, s);
  return cudaGetLastError();
}

cudaError_t launch_transd_project(const float* ent, int ent_dim, const float* s, const float* rel_proj_row,
                                  int64_t n_rows, int rel_dim, float* out, cudaStream_t stream) {
  const long long total = (long long)n_rows * rel_dim;
  if (total <= 0) return cudaSuccess;
  const long long want = blocks_for(total, 256);
  const unsigned blocks = (unsigned)(want > 132LL * 16 ? 132LL * 16 : want);   // grid-stride past 16 per SM
  transd_project_kernel<<<blocks, 256, 0, stream>>>(ent, ent_dim, s, rel_proj_row, total, rel_dim, out);
  return cudaGetLastError();
}

cudaError_t launch_finalize(const int32_t* raw, const int32_t* sub, int64_t n, int64_t* ranks,
                            int64_t* filt_ranks, cudaStream_t stream) {
  if (n <= 0) return cudaSuccess;
  finalize_kernel<<<blocks_for(n, 256), 256, 0, stream>>>(raw, sub, n, ranks, filt_ranks);
  return cudaGetLastError();
}

}  // namespace kge
