// Device-side score arithmetic shared by every kernel (dense scan, sparse pair scorer).
// One (query, candidate) score = "element term" per embedding index, reduced by replaying
// a Schedule (schedule.h).  Every operation is an explicitly rounded intrinsic so the
// compiler can neither contract mul+add into fma nor reassociate: bit-equality between the
// dense scan, the true-score pass and the filter pass -- and with ATen's CPU kernels --
// rests on that.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "schedule.h"

namespace kge {

// Element kinds: how one term is formed from the query planes q[] and candidate planes c[].
enum ElemKind : int {
  EL_DOT1 = 0,     // q0*c0                      DistMult bilinear.py:235,240 ; RESCAL :109,114
  EL_DOT2 = 1,     // q0*c0 + q1*c1              ComplEx  bilinear.py:514-515, 521-522
  EL_L1_TAIL = 2,  // |q0 - c0|                  interfaces.py:253-254 + dissimilarities.py:16
  EL_L1_HEAD = 3,  // |(c0 + q0) - q1|           interfaces.py:258-260 + dissimilarities.py:16
  EL_L2_TAIL = 4,  // (q0 - c0)^2                interfaces.py:253-254 + dissimilarities.py:25
  EL_L2_HEAD = 5,  // ((c0 + q0) - q1)^2         interfaces.py:258-260 + dissimilarities.py:25
  EL_ROT = 6,      // sqrt((q0-c0)^2+(q1-c1)^2)  oracle RotatE restatement
  EL_DOT_MID = 7,  // (q0*c0)*q1                 DistMult relation prediction, bilinear.py:243-245
  // TorusE (translation.py:655-767), x = q0 - c0 (tail) or (c0 + q0) - q1 (head):
  EL_TL1_TAIL = 8,   // 2*min(|x|, 1-|x|)         dissimilarities.py:28-34
  EL_TL1_HEAD = 9,
  EL_TL2_TAIL = 10,  // 4*min(x^2, 1-x^2)         dissimilarities.py:37-43
  EL_TL2_HEAD = 11,
  // Analogy (bilinear.py:694-712), three planes (scalar, real, imaginary) of equal width:
  EL_DOT3 = 12,      // (q0*c0 + qm*cm) + q1*c1   (qm / cm: the middle plane)
  EL_COUNT = 13
};

template <int EL> struct ElemTraits;
template <> struct ElemTraits<EL_DOT1> { static constexpr int QW = 1, CW = 1, RED = RED_SUM; };
template <> struct ElemTraits<EL_DOT2> { static constexpr int QW = 2, CW = 2, RED = RED_SUM; };
template <> struct ElemTraits<EL_L1_TAIL> { static constexpr int QW = 1, CW = 1, RED = RED_SEQ; };
template <> struct ElemTraits<EL_L1_HEAD> { static constexpr int QW = 2, CW = 1, RED = RED_SEQ; };
template <> struct ElemTraits<EL_L2_TAIL> { static constexpr int QW = 1, CW = 1, RED = RED_NORM2; };
template <> struct ElemTraits<EL_L2_HEAD> { static constexpr int QW = 2, CW = 1, RED = RED_NORM2; };
template <> struct ElemTraits<EL_ROT> { static constexpr int QW = 2, CW = 2, RED = RED_SUM; };
template <> struct ElemTraits<EL_DOT_MID> { static constexpr int QW = 2, CW = 1, RED = RED_SUM; };
template <> struct ElemTraits<EL_TL1_TAIL> { static constexpr int QW = 1, CW = 1, RED = RED_SUM; };
template <> struct ElemTraits<EL_TL1_HEAD> { static constexpr int QW = 2, CW = 1, RED = RED_SUM; };
template <> struct ElemTraits<EL_TL2_TAIL> { static constexpr int QW = 1, CW = 1, RED = RED_SUM; };
template <> struct ElemTraits<EL_TL2_HEAD> { static constexpr int QW = 2, CW = 1, RED = RED_SUM; };
template <> struct ElemTraits<EL_DOT3> { static constexpr int QW = 3, CW = 3, RED = RED_SUM; };

// torch.min(a, b) element-wise: NaN propagates (ATen minimum), otherwise the smaller
__device__ __forceinline__ float aten_min(float a, float b) { return (a != a || a < b) ? a : b; }

// For the L2 kinds returns the difference x (the caller squares it, fused or not); for all
// other kinds returns the finished term.  q0 / c0 = first plane, q1 / c1 = LAST plane, qm / cm =
// middle plane (three-plane kinds only).
template <int EL>
__device__ __forceinline__ float elem_value(float q0, float q1, float c0, float c1, float qm = 0.f,
                                            float cm = 0.f) {
  if constexpr (EL == EL_DOT1) {
    return __fmul_rn(q0, c0);
  } else if constexpr (EL == EL_DOT2) {
    return __fadd_rn(__fmul_rn(q0, c0), __fmul_rn(q1, c1));
  } else if constexpr (EL == EL_DOT3) {
    return __fadd_rn(__fadd_rn(__fmul_rn(q0, c0), __fmul_rn(qm, cm)), __fmul_rn(q1, c1));
  } else if constexpr (EL == EL_L1_TAIL) {
    return fabsf(__fsub_rn(q0, c0));
  } else if constexpr (EL == EL_L1_HEAD) {
    return fabsf(__fsub_rn(__fadd_rn(c0, q0), q1));
  } else if constexpr (EL == EL_L2_TAIL) {
    return __fsub_rn(q0, c0);
  } else if constexpr (EL == EL_L2_HEAD) {
    return __fsub_rn(__fadd_rn(c0, q0), q1);
  } else if constexpr (EL == EL_DOT_MID) {
    return __fmul_rn(__fmul_rn(q0, c0), q1);
  } else if constexpr (EL == EL_TL1_TAIL || EL == EL_TL1_HEAD) {
    // 2 * min(abs(a - b), 1 - abs(a - b)) summed: the factor is applied per element in the
    // reference (exact in fp32), before the cascade sum
    const float x = EL == EL_TL1_TAIL ? __fsub_rn(q0, c0) : __fsub_rn(__fadd_rn(c0, q0), q1);
    const float ax = fabsf(x);
    return __fmul_rn(2.f, aten_min(ax, __fsub_rn(1.f, ax)));
  } else if constexpr (EL == EL_TL2_TAIL || EL == EL_TL2_HEAD) {
    const float x = EL == EL_TL2_TAIL ? __fsub_rn(q0, c0) : __fsub_rn(__fadd_rn(c0, q0), q1);
    const float x2 = __fmul_rn(x, x);
    return __fmul_rn(4.f, aten_min(x2, __fsub_rn(1.f, x2)));
  } else {  // EL_ROT
    const float dr = __fsub_rn(q0, c0);
    const float di = __fsub_rn(q1, c1);
    return __fsqrt_rn(__fadd_rn(__fmul_rn(dr, dr), __fmul_rn(di, di)));
  }
}

// Approximate element for the bound-and-refine scan (EL_ROT): fused multiply-add and the
// hardware's approximate square root (MUFU), any association -- the result only has to be within
// a known relative error of the exactly rounded one.
__device__ __forceinline__ float elem_rot_fast(float q0, float q1, float c0, float c1) {
  const float dr = q0 - c0, di = q1 - c1;
  float r;
  // .ftz: a squared modulus below 2^-126 reads as 0 -- an absolute error below 1.1e-19 per term,
  // carried by the scan's thresholds (ScanParams::abs_eps)
#if defined(__CUDACC__)
  asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(fmaf(di, di, dr * dr)));
#else
  r = sqrtf(fmaf(di, di, dr * dr));  // host build of this header (tests/host_arith.cpp) only
#endif
  return r;
}

template <int EL>
__device__ __forceinline__ constexpr bool elem_is_l2() {
  return EL == EL_L2_TAIL || EL == EL_L2_HEAD;
}

// The code byte that needs no combine step and is by far the most frequent one.
template <int EL>
__device__ __forceinline__ constexpr uint8_t fast_code() {
  return ElemTraits<EL>::RED == RED_SEQ ? SC_MODE_T : SC_MODE_A;
}

// Registers of one running (query, candidate) reduction.
struct Acc {
  float a, a1, p, t;
};

__device__ __forceinline__ void acc_reset(Acc& r) { r.a = r.a1 = r.p = r.t = 0.f; }

// Fast path: position whose code is fast_code<EL>().
template <int EL>
__device__ __forceinline__ void acc_step_fast(Acc& r, float q0, float q1, float c0, float c1,
                                              float qm = 0.f, float cm = 0.f) {
  float v = elem_value<EL>(q0, q1, c0, c1, qm, cm);
  if constexpr (elem_is_l2<EL>()) v = __fmul_rn(v, v);
  if constexpr (ElemTraits<EL>::RED == RED_SEQ)
    r.t = __fadd_rn(r.t, v);
  else
    r.a = __fadd_rn(r.a, v);
}

// General path for ONE pair (sparse pair scorer).  `code` is uniform across the warp there too.
template <int EL, bool CASC>
__device__ __forceinline__ void acc_step(Acc& r, uint8_t code, float q0, float q1, float c0,
                                         float c1, float qm = 0.f, float cm = 0.f) {
  const float v = elem_value<EL>(q0, q1, c0, c1, qm, cm);
  const uint8_t mode = code & SC_MODE_MASK;
  if constexpr (elem_is_l2<EL>()) {
    if (mode == SC_MODE_A)
      r.a = __fadd_rn(r.a, __fmul_rn(v, v));
    else if (mode == SC_MODE_T)
      r.t = __fadd_rn(r.t, __fmul_rn(v, v));
    else
      r.t = __fmaf_rn(v, v, r.t);
  } else {
    if (mode == SC_MODE_A)
      r.a = __fadd_rn(r.a, v);
    else
      r.t = __fadd_rn(r.t, v);
  }
  if constexpr (CASC) {
    if (code & SC_CASC1) { r.a1 = __fadd_rn(r.a1, r.a); r.a = 0.f; }
    if (code & SC_FOLD1) { r.a = __fadd_rn(r.a, r.a1); r.a1 = 0.f; }
  }
  if (code & SC_P_SET) { r.p = r.a; r.a = 0.f; }
  if (code & SC_P_ADD) { r.p = __fadd_rn(r.p, r.a); r.a = 0.f; }
  if (code & SC_T_ADD_P) { r.t = __fadd_rn(r.t, r.p); }
  if (code & SC_T_ADD_A) { r.t = __fadd_rn(r.t, r.a); r.a = 0.f; }
}

// The same step split for register tiles: the element part for one pair under a given
// (uniform) mode, and the combine part for one pair under a given (uniform) op.  The dense
// scan hoists the uniform tests out of its pair loops, so no per-pair selects are generated.
template <int EL>
__device__ __forceinline__ void acc_elem_mode(Acc& r, uint8_t mode, float q0, float q1, float c0,
                                              float c1, float qm = 0.f, float cm = 0.f) {
  const float v = elem_value<EL>(q0, q1, c0, c1, qm, cm);
  if constexpr (elem_is_l2<EL>()) {
    if (mode == SC_MODE_A)
      r.a = __fadd_rn(r.a, __fmul_rn(v, v));
    else if (mode == SC_MODE_T)
      r.t = __fadd_rn(r.t, __fmul_rn(v, v));
    else
      r.t = __fmaf_rn(v, v, r.t);
  } else {
    if (mode == SC_MODE_A)
      r.a = __fadd_rn(r.a, v);
    else
      r.t = __fadd_rn(r.t, v);
  }
}

__device__ __forceinline__ void acc_casc1(Acc& r) { r.a1 = __fadd_rn(r.a1, r.a); r.a = 0.f; }
__device__ __forceinline__ void acc_fold1(Acc& r) { r.a = __fadd_rn(r.a, r.a1); r.a1 = 0.f; }
__device__ __forceinline__ void acc_p_set(Acc& r) { r.p = r.a; r.a = 0.f; }
__device__ __forceinline__ void acc_p_add(Acc& r) { r.p = __fadd_rn(r.p, r.a); r.a = 0.f; }
__device__ __forceinline__ void acc_t_add_p(Acc& r) { r.t = __fadd_rn(r.t, r.p); }
__device__ __forceinline__ void acc_t_add_a(Acc& r) { r.t = __fadd_rn(r.t, r.a); r.a = 0.f; }

// Reduction result -> score, with the reference's sign and the L2 sqrt-then-square
// (dissimilarities.py:25 computes norm(p=2)**2; interfaces.py:254,260 negate).
template <int EL>
__device__ __forceinline__ float acc_finish(const Acc& r) {
  if constexpr (EL == EL_DOT1 || EL == EL_DOT2 || EL == EL_DOT3 || EL == EL_DOT_MID) {
    return r.t;
  } else if constexpr (elem_is_l2<EL>()) {
    const float n = __fsqrt_rn(r.t);
    return -__fmul_rn(n, n);
  } else {
    return -r.t;
  }
}

// Exact score of one pair in NATURAL index order.  Same arithmetic as replaying the schedule
// (every chain of the ATen reduction receives the same terms in the same order, chains are
// combined in the same order) but the embedding index runs 0, 1, 2, ... so each thread streams
// its two rows sequentially instead of revisiting every 32-byte sector eight times; the chain
// accumulators live in registers (8 for the L2 norm, 32 (+32 cascade) for the cascade sum).
template <int EL>
__device__ __forceinline__ float elem_at(const float* q0, const float* q1, const float* c0,
                                         const float* c1, int k, const float* qm = nullptr,
                                         const float* cm = nullptr) {
  if constexpr (ElemTraits<EL>::CW == 3)
    return elem_value<EL>(q0[k], q1[k], c0[k], c1[k], qm[k], cm[k]);
  else
    return elem_value<EL>(q0[k], q1[k], c0[k], c1[k]);
}

template <int EL>
__device__ float pair_score_natural(int dim, const float* __restrict__ q0, const float* __restrict__ q1,
                                    const float* __restrict__ c0, const float* __restrict__ c1,
                                    const float* __restrict__ qm = nullptr,
                                    const float* __restrict__ cm = nullptr) {
  if constexpr (ElemTraits<EL>::RED == RED_NORM2) {
    const int main_len = dim - dim % 8;
    float acc[8];
#pragma unroll
    for (int l = 0; l < 8; ++l) acc[l] = 0.f;
    for (int k = 0; k < main_len; k += 8) {
#pragma unroll
      for (int l = 0; l < 8; ++l) {
        const float x = elem_at<EL>(q0, q1, c0, c1, k + l, qm, cm);
        acc[l] = __fadd_rn(acc[l], __fmul_rn(x, x));
      }
    }
    float t = 0.f;
    if (main_len > 0) {
#pragma unroll
      for (int l = 0; l < 8; ++l) t = __fadd_rn(t, acc[l]);
    }
    int k = main_len;
    for (; k + 4 <= dim; k += 4) {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float x = elem_at<EL>(q0, q1, c0, c1, k + j, qm, cm);
        t = __fadd_rn(t, __fmul_rn(x, x));
      }
    }
    for (; k < dim; ++k) {
      const float x = elem_at<EL>(q0, q1, c0, c1, k, qm, cm);
      t = __fmaf_rn(x, x, t);
    }
    Acc r; r.a = r.a1 = r.p = 0.f; r.t = t;
    return acc_finish<EL>(r);
  } else {  // RED_SUM
    float t = 0.f;
    if (dim >= 8) {
      const int vec_size = dim / 8, rows = vec_size / 4;
      const bool casc = rows >= 16;
      for (int k = vec_size * 8; k < dim; ++k) t = __fadd_rn(t, elem_at<EL>(q0, q1, c0, c1, k, qm, cm));
      float acc[4][8], acc1[4][8];
#pragma unroll
      for (int m = 0; m < 4; ++m)
#pragma unroll
        for (int l = 0; l < 8; ++l) { acc[m][l] = 0.f; acc1[m][l] = 0.f; }
      for (int i = 0; i < rows; ++i) {
        const int k0 = i * 32;
#pragma unroll
        for (int m = 0; m < 4; ++m)
#pragma unroll
          for (int l = 0; l < 8; ++l)
            acc[m][l] = __fadd_rn(acc[m][l], elem_at<EL>(q0, q1, c0, c1, k0 + m * 8 + l, qm, cm));
        if (((i + 1) & 15) == 0) {
#pragma unroll
          for (int m = 0; m < 4; ++m)
#pragma unroll
            for (int l = 0; l < 8; ++l) { acc1[m][l] = __fadd_rn(acc1[m][l], acc[m][l]); acc[m][l] = 0.f; }
        }
      }
      if (casc) {
#pragma unroll
        for (int m = 0; m < 4; ++m)
#pragma unroll
          for (int l = 0; l < 8; ++l) acc[m][l] = __fadd_rn(acc[m][l], acc1[m][l]);
      }
      for (int j = rows * 4; j < vec_size; ++j) {
#pragma unroll
        for (int l = 0; l < 8; ++l) acc[0][l] = __fadd_rn(acc[0][l], elem_at<EL>(q0, q1, c0, c1, j * 8 + l, qm, cm));
      }
#pragma unroll
      for (int l = 0; l < 8; ++l) {
        float pl = acc[0][l];
        if (rows > 0) {
#pragma unroll
          for (int m = 1; m < 4; ++m) pl = __fadd_rn(pl, acc[m][l]);
        }
        t = __fadd_rn(t, pl);
      }
    } else {  // one lane: 4 interleaved chains, leftovers to chain 0
      const int rows = dim / 4;
      float acc[4] = {0.f, 0.f, 0.f, 0.f};
      for (int i = 0; i < rows; ++i) {
#pragma unroll
        for (int m = 0; m < 4; ++m) acc[m] = __fadd_rn(acc[m], elem_at<EL>(q0, q1, c0, c1, i * 4 + m, qm, cm));
      }
      for (int k = rows * 4; k < dim; ++k) acc[0] = __fadd_rn(acc[0], elem_at<EL>(q0, q1, c0, c1, k, qm, cm));
      float pl = acc[0];
      if (rows > 0) {
#pragma unroll
        for (int m = 1; m < 4; ++m) pl = __fadd_rn(pl, acc[m]);
      }
      t = __fadd_rn(t, pl);
    }
    Acc r; r.a = r.a1 = r.p = 0.f; r.t = t;
    return acc_finish<EL>(r);
  }
}

// RESCAL query preparation, one output component (bilinear.py:108 `matmul(r, t.view(b, d, 1))`,
// :113 `matmul(h.view(b, 1, d), r)`): the reference's batched matmul runs in oneMKL (ATen bmm ->
// cblas_sgemm_batch) for d >= 20 and in ATen's own scalar loop (baddbmm_cpu_kernel, mul and add
// rounded separately) below that (contraction * rows * cols < 400).  The summation ORDER below was
// recovered by probing torch 2.11 / oneMKL 2024.2 (AVX-512 code path) with absorption tests
// (2^25, 1, -2^25 at three positions of the contraction) and confirmed bit for bit on random data
// for every d in 1..512 and for d up to 8191 at and around every K-block boundary
// (tests/test_host_arith.py replays this very function on the host):
//   tail  q_j = sum_k h_k M[k][j], columns j < 16*floor(d/16) (full 16-lane vectors):
//           per chunk of 8 k:  y = fma(h6,M6,y); y = fma(h4,M4,y); y += fma(h5,M5,h7*M7);
//                              y += fma(h0,M0,h2*M2) + fma(h1,M1,h3*M3);   then a plain fma chain
//           over the d % 8 leftover k;  remainder columns: one fma chain over all k
//   head  q_j = sum_k M[j][k] t_k: one fma chain over k for d <= 384; beyond, one fma chain per
//           K-block of 384 from k = 0 while more than 768 terms remain, then the last a..d-1
//           (385..768 terms) as two chains [a, m) and [m, d), m = a + ceil((d - a)/2); the chains
//           are added left to right (d = 1000: [0,384) [384,692) [692,1000); d <= 768: the halves)
// `vec` = h (tail) or t (head); M row-major (d, d).  A batch of exactly ONE fact takes a different
// MKL path in the reference (sgemv with alignment-dependent peeling, not reproducible): documented.
__device__ __forceinline__ float rescal_query_component(bool tail, int d, int j, const float* __restrict__ vec,
                                                        const float* __restrict__ M) {
  float acc = 0.f;
  if (tail) {
    const float* col = M + j;  // M[k][j] = col[k * d]
    if (d < 20) {
      for (int k = 0; k < d; ++k) acc = __fadd_rn(acc, __fmul_rn(vec[k], col[(size_t)k * d]));
    } else if (j < (d / 16) * 16) {
      int k = 0;
      for (; k + 8 <= d; k += 8) {
        const float* c = col + (size_t)k * d;
        acc = __fmaf_rn(vec[k + 6], c[(size_t)6 * d], acc);
        acc = __fmaf_rn(vec[k + 4], c[(size_t)4 * d], acc);
        acc = __fadd_rn(acc, __fmaf_rn(vec[k + 5], c[(size_t)5 * d], __fmul_rn(vec[k + 7], c[(size_t)7 * d])));
        const float e = __fmaf_rn(vec[k], c[0], __fmul_rn(vec[k + 2], c[(size_t)2 * d]));
        const float o = __fmaf_rn(vec[k + 1], c[d], __fmul_rn(vec[k + 3], c[(size_t)3 * d]));
        acc = __fadd_rn(acc, __fadd_rn(e, o));
      }
      for (; k < d; ++k) acc = __fmaf_rn(vec[k], col[(size_t)k * d], acc);
    } else {
      for (int k = 0; k < d; ++k) acc = __fmaf_rn(vec[k], col[(size_t)k * d], acc);
    }
  } else {
    const float* row = M + (size_t)j * d;
    if (d < 20) {
      for (int k = 0; k < d; ++k) acc = __fadd_rn(acc, __fmul_rn(row[k], vec[k]));
    } else if (d <= 384) {
      for (int k = 0; k < d; ++k) acc = __fmaf_rn(row[k], vec[k], acc);
    } else {
      int a = 0;
      for (; d - a > 768; a += 384) {   // K-blocks of 384 while more than 768 terms remain
        float c = 0.f;
        for (int k = a; k < a + 384; ++k) c = __fmaf_rn(row[k], vec[k], c);
        acc = a == 0 ? c : __fadd_rn(acc, c);
      }
      const int mid = a + (d - a + 1) / 2;   // the last 385..768 terms: two chains
      float c0 = 0.f, c1 = 0.f;
      for (int k = a; k < mid; ++k) c0 = __fmaf_rn(row[k], vec[k], c0);
      for (int k = mid; k < d; ++k) c1 = __fmaf_rn(row[k], vec[k], c1);
      acc = __fadd_rn(a == 0 ? c0 : __fadd_rn(acc, c0), c1);
    }
  }
  return acc;
}

// TransH's projection of an entity row e on the hyperplane of normal w (translation.py:279-281,
// evaluate_projections):  P[k] = fl(e[k] - fl(nc * w[k]))  with  nc = (e * w).sum()  summed in ATen's
// inner-dimension order (pair_score_natural / pair_score_chains of EL_DOT1 give that sum).  The inputs
// are the raw ent_emb / norm_vect rows: the reference does not re-normalise them there.
__device__ __forceinline__ float transh_project_elem(float e, float nc, float w) {
  return __fsub_rn(e, __fmul_rn(nc, w));
}

// TransD's projection of entity coordinate j < rel_emb_dim under relation r (translation.py:645-646,
// evaluate_projectionss):  P[j] = fl(fl(s * rp[j]) + e[j])  with  s = (ent_proj_vect[e] * ent_emb[e]).sum()
// over ent_emb_dim, summed in ATen's inner-dimension order (EL_DOT1 of pair_score_natural / pair_score_chains)
// and rp = rel_proj_vect[r].  Two roundings: the reference multiplies, then adds, and fuses nothing.
__device__ __forceinline__ float transd_project_elem(float e, float s, float rp) {
  return __fadd_rn(__fmul_rn(s, rp), e);
}

// Exact adjudication of the near-tie band (the list is kept as one region per CTA of the scan).
// Chain-parallel: the independent chains of the ATen reduction are spread over the lanes of a
// warp -- 8 lanes per pair for the L2 norm (4 pairs per warp), 32 lanes per pair for the
// cascade sum -- so each step reads 32 / 128 contiguous bytes of the two rows; chains are then
// combined through shuffles in exactly the schedule's order.  Same bits as pair_score_natural.
template <int EL>
__device__ __forceinline__ float pair_score_chains(int dim, const float* __restrict__ q0,
                                                   const float* __restrict__ q1,
                                                   const float* __restrict__ c0,
                                                   const float* __restrict__ c1, int lane,
                                                   const float* __restrict__ qm = nullptr,
                                                   const float* __restrict__ cm = nullptr) {
  if constexpr (ElemTraits<EL>::RED == RED_NORM2) {
    const int l8 = lane & 7, g8 = lane & 24;  // lane of the norm, first lane of this pair's group
    const int main_len = dim - dim % 8;
    float acc = 0.f;
    for (int k = l8; k < main_len; k += 8) {
      const float x = elem_at<EL>(q0, q1, c0, c1, k, qm, cm);
      acc = __fadd_rn(acc, __fmul_rn(x, x));
    }
    float t = 0.f;
#pragma unroll
    for (int l = 0; l < 8; ++l) {
      const float v = __shfl_sync(0xffffffffu, acc, g8 + l);
      if (main_len > 0) t = __fadd_rn(t, v);
    }
    int k = main_len;
    for (; k + 4 <= dim; k += 4) {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float x = elem_at<EL>(q0, q1, c0, c1, k + j, qm, cm);
        t = __fadd_rn(t, __fmul_rn(x, x));
      }
    }
    for (; k < dim; ++k) {
      const float x = elem_at<EL>(q0, q1, c0, c1, k, qm, cm);
      t = __fmaf_rn(x, x, t);
    }
    Acc r; r.a = r.a1 = r.p = 0.f; r.t = t;
    return acc_finish<EL>(r);
  } else {  // RED_SUM, dim >= 8: lane = 8 m + l owns chain (row m, lane l)
    const int vec_size = dim / 8, rows = vec_size / 4;
    float acc = 0.f, acc1 = 0.f;
    for (int i = 0; i < rows; ++i) {
      acc = __fadd_rn(acc, elem_at<EL>(q0, q1, c0, c1, i * 32 + lane, qm, cm));
      if (((i + 1) & 15) == 0) { acc1 = __fadd_rn(acc1, acc); acc = 0.f; }
    }
    if (rows >= 16) acc = __fadd_rn(acc, acc1);
    if (lane < 8)
      for (int j = rows * 4; j < vec_size; ++j) acc = __fadd_rn(acc, elem_at<EL>(q0, q1, c0, c1, j * 8 + lane, qm, cm));
    const int l = lane & 7;
    float pl = __shfl_sync(0xffffffffu, acc, l);
#pragma unroll
    for (int m = 1; m < 4; ++m) {
      const float v = __shfl_sync(0xffffffffu, acc, 8 * m + l);
      if (rows > 0) pl = __fadd_rn(pl, v);
    }
    float t = 0.f;
    for (int k = vec_size * 8; k < dim; ++k) t = __fadd_rn(t, elem_at<EL>(q0, q1, c0, c1, k, qm, cm));
#pragma unroll
    for (int ll = 0; ll < 8; ++ll) t = __fadd_rn(t, __shfl_sync(0xffffffffu, pl, ll));
    Acc r; r.a = r.a1 = r.p = 0.f; r.t = t;
    return acc_finish<EL>(r);
  }
}


}  // namespace kge
