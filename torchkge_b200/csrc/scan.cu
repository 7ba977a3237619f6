// Dense rank scan: the kernel that replaces inference_scoring_function + get_rank
// (torchkge models/interfaces.py:240-260, models/bilinear.py:98-121,224-245,501-528,
// utils/operations.py:37-61) for one side of a batch of test triples.
//
// Shape of the work: S[q][c] = reduce_k f(Q[q][k], E[c][k]) over n_q queries x n_rows
// candidates x dim, of which only  #{c : S[q][c] >= s_true[q]}  per query is kept.  With
// tens of thousands of queries sharing every streamed candidate tile the kernel is bound by
// fp32 issue, not by HBM, so it is organised like an SGEMM: a persistent CTA per SM walks
// (query tile, candidate tile) pairs; one elected thread streams schedule-ordered k-chunks of
// both operands into a shared-memory ring with 1-D bulk async copies (UBLKCP) signalled on
// mbarriers, two stages ahead; all warps hold a register tile of running reductions per thread.  Both
// operands are pre-laid out k-major ("packed") so every shared-memory read is a conflict-free
// 128-bit load and the reduction schedule is walked front to back.  Positions that need a
// combine step are flagged in a per-stage bit mask, so the common positions run in branch-free
// unrolled runs.
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "kernels.h"
#include "ptx.cuh"

namespace kge {

namespace {

constexpr int KC = SCAN_KC;  // schedule positions per pipeline stage (one 32-bit special mask)
constexpr int STAGES = 3;
constexpr int TQ = 4;   // queries per thread

// G = groups of 4 candidates per thread (thread tile 4 x 4G); consumer warps = 16 / G.
template <int EL, int G>
struct Cfg {
  static constexpr int QW = ElemTraits<EL>::QW;
  static constexpr int CW = ElemTraits<EL>::CW;
  static constexpr int TC = 4 * G;
  static constexpr int WARPS_C = TILE_C / (32 * G);      // warps along candidates
  static constexpr int WARPS_Q = TILE_Q / 16;            // warps along queries
  static constexpr int CONSUMER_WARPS = WARPS_C * WARPS_Q;
  static constexpr int THREADS = CONSUMER_WARPS * 32;
  static constexpr int C_FLOATS = KC * CW * TILE_C;
  static constexpr int Q_FLOATS = KC * QW * TILE_Q;
  static constexpr int STAGE_FLOATS = C_FLOATS + Q_FLOATS;
  static constexpr size_t SMEM_BYTES =
      (size_t)STAGES * STAGE_FLOATS * sizeof(float) + 2 * STAGES * sizeof(uint64_t);
};

// APPROX (EL_ROT): bound-and-refine form.  The element is evaluated with FMA + MUFU.SQRT and
// summed in two levels (per 32-position stage, then across stages: depth <= 32 + dim/32), which is
// within  rel_eps * |s|  of the exactly rounded ATen-order score because every term is >= 0; pairs
// that the approximate score cannot place on one side of s_true go to the near-tie list and are
// re-scored exactly (tc.cu: recheck_kernel<EL_ROT>).  The exact form pays ~16 fp32 instructions
// per element for the correctly rounded sqrt; this one 6 + one MUFU.
template <int EL, bool CASC, int G, bool APPROX>
__global__ void __launch_bounds__(Cfg<EL, G>::THREADS, 1)
    scan_kernel(const __grid_constant__ ScanParams p) {
  using L = Cfg<EL, G>;
  constexpr int QW = L::QW, CW = L::CW, TC = L::TC;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  float* stage_base = reinterpret_cast<float*>(smem_raw);
  uint64_t* full_bar =
      reinterpret_cast<uint64_t*>(smem_raw + (size_t)STAGES * L::STAGE_FLOATS * sizeof(float));
  uint64_t* empty_bar = full_bar + STAGES;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int dim = p.dim;
  const int n_kc = (dim + KC - 1) / KC;
  const long long total_tiles = (long long)p.n_qt * (long long)p.n_ct;

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      ptx::mbar_init(&full_bar[s], 1);
      ptx::mbar_init(&empty_bar[s], L::CONSUMER_WARPS);
    }
    ptx::fence_mbar_init();
  }
  __syncthreads();

  // ---- producer duty: one elected thread (lane 0 of the last warp) keeps the ring STAGES-1
  // stages ahead of the consumers.  Stage number g counts (tile, k-chunk) pairs of this CTA.
  const long long my_tiles = (total_tiles - blockIdx.x + gridDim.x - 1) / gridDim.x;
  const long long total_stages = my_tiles * n_kc;
  const bool is_producer = (warp == L::CONSUMER_WARPS - 1) && (lane == 0);
  long long prod_tile = blockIdx.x;  // tile of the next stage to issue
  int prod_kc = 0;
  long long prod_g = 0;
  auto issue_next = [&]() {
    const int slot = (int)(prod_g % STAGES);
    const long long use = prod_g / STAGES;
    if (use > 0) ptx::mbar_wait(&empty_bar[slot], (uint32_t)((use - 1) & 1));
    const long long qt = prod_tile / p.n_ct;
    const long long ct = prod_tile - qt * p.n_ct;
    const int kn = min(KC, dim - prod_kc * KC);
    float* sc = stage_base + (size_t)slot * L::STAGE_FLOATS;
    float* sq = sc + L::C_FLOATS;
    const uint32_t cbytes = (uint32_t)kn * CW * TILE_C * sizeof(float);
    const uint32_t qbytes = (uint32_t)kn * QW * TILE_Q * sizeof(float);
    ptx::mbar_arrive_expect_tx(&full_bar[slot], cbytes + qbytes);
    ptx::bulk_g2s(sc, p.packed + ((size_t)ct * dim + (size_t)prod_kc * KC) * (CW * TILE_C), cbytes,
                  &full_bar[slot]);
    ptx::bulk_g2s(sq, p.qpacked + ((size_t)qt * dim + (size_t)prod_kc * KC) * (QW * TILE_Q), qbytes,
                  &full_bar[slot]);
    ++prod_g;
    if (++prod_kc == n_kc) { prod_kc = 0; prod_tile += gridDim.x; }
  };
  if (is_producer)
    for (int g = 0; g < STAGES - 1 && prod_g < total_stages; ++g) issue_next();

  // -------------------------------- consumer warps --------------------------------
  const int wq = warp / L::WARPS_C, wc = warp % L::WARPS_C;
  const int tq = lane >> 3, tc = lane & 7;  // 4 x 8 threads per warp
  const int q_off = wq * 16 + tq * TQ;
  const int c_off = wc * (32 * G) + tc * 4;  // group g adds 32 * g

  int stage = 0;
  uint32_t phase = 0;
  long long cur_qt = -1;
  float st[TQ];
  float t_hi[TQ], t_lo[TQ];  // APPROX only
  int cnt[TQ];
#pragma unroll
  for (int i = 0; i < TQ; ++i) { st[i] = 0.f; cnt[i] = 0; t_hi[i] = t_lo[i] = 0.f; }

  auto flush_counts = [&](long long qt) {
    if (p.counts == nullptr || qt < 0) return;
#pragma unroll
    for (int i = 0; i < TQ; ++i) {
      int v = cnt[i];
      v += __shfl_xor_sync(0xffffffffu, v, 1);
      v += __shfl_xor_sync(0xffffffffu, v, 2);
      v += __shfl_xor_sync(0xffffffffu, v, 4);
      const long long q = qt * TILE_Q + q_off + i;
      if (tc == 0 && v != 0 && q < p.n_q) atomicAdd(&p.counts[q], v);
      cnt[i] = 0;
    }
  };

  for (long long tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
    const long long qt = tile / p.n_ct;
    const long long ct = tile - qt * p.n_ct;
    if (qt != cur_qt) {
      flush_counts(cur_qt);
      cur_qt = qt;
#pragma unroll
      for (int i = 0; i < TQ; ++i) st[i] = p.s_true[qt * TILE_Q + q_off + i];
      if constexpr (APPROX) {
        // scores are <= 0 (minus a sum of moduli), |s_exact - s~| <= g |s~|:
        //   s~ > st / (1 + g)  =>  s > st ;  s~ < st / (1 - g)  =>  s < st   (directed rounding)
#pragma unroll
        for (int i = 0; i < TQ; ++i) {
          t_hi[i] = __fadd_ru(__fdiv_ru(st[i], 1.f + p.rel_eps), p.abs_eps);
          t_lo[i] = __fadd_rd(__fdiv_rd(st[i], 1.f - p.rel_eps), -p.abs_eps);
          if (st[i] > 0.f) { t_hi[i] = INFINITY; t_lo[i] = -INFINITY; }  // cannot happen; stay exact
        }
      }
    }

    Acc acc[TQ][TC];
#pragma unroll
    for (int i = 0; i < TQ; ++i)
#pragma unroll
      for (int j = 0; j < TC; ++j) acc_reset(acc[i][j]);

    for (int kc = 0; kc < n_kc; ++kc) {
      const int kn = min(KC, dim - kc * KC);
      const uint32_t special = p.mask[kc];
      if (is_producer && prod_g < total_stages) issue_next();
      ptx::mbar_wait(&full_bar[stage], phase);
      const float* sc = stage_base + (size_t)stage * L::STAGE_FLOATS + c_off;
      const float* sq = stage_base + (size_t)stage * L::STAGE_FLOATS + L::C_FLOATS + q_off;

      auto load_operands = [&](int kk, float (&qv)[QW][TQ], float (&cv)[CW][TC]) {
#pragma unroll
        for (int w = 0; w < QW; ++w) {
          const float4 v = *reinterpret_cast<const float4*>(sq + (kk * QW + w) * TILE_Q);
          qv[w][0] = v.x; qv[w][1] = v.y; qv[w][2] = v.z; qv[w][3] = v.w;
        }
#pragma unroll
        for (int w = 0; w < CW; ++w)
#pragma unroll
          for (int g = 0; g < G; ++g) {
            const float4 v = *reinterpret_cast<const float4*>(sc + (kk * CW + w) * TILE_C + 32 * g);
            cv[w][4 * g + 0] = v.x; cv[w][4 * g + 1] = v.y;
            cv[w][4 * g + 2] = v.z; cv[w][4 * g + 3] = v.w;
          }
      };

      // One schedule position: ordinary element step for all pairs, then -- only if the
      // position is flagged in the stage mask -- the combine steps, each behind a uniform test.
      // Operands of the NEXT position are fetched before the current one is consumed (explicit
      // two-deep register pipeline; the loop is unrolled by two so no register copies remain).
#define KGE_FOR_PAIRS(stmt)                       \
  _Pragma("unroll") for (int i = 0; i < TQ; ++i)  \
  _Pragma("unroll") for (int c = 0; c < TC; ++c) { stmt; }
      auto consume = [&](int kk, float (&qv)[QW][TQ], float (&cv)[CW][TC]) {
        if (!((special >> kk) & 1u)) {
          KGE_FOR_PAIRS(acc_step_fast<EL>(acc[i][c], qv[0][i], qv[QW - 1][i], cv[0][c], cv[CW - 1][c], qv[QW / 2][i], cv[CW / 2][c]))
        } else {
          const uint8_t code = p.code[kc * KC + kk];
          const uint8_t mode = code & SC_MODE_MASK;
          if (mode == SC_MODE_A) {
            KGE_FOR_PAIRS(acc_elem_mode<EL>(acc[i][c], SC_MODE_A, qv[0][i], qv[QW - 1][i], cv[0][c], cv[CW - 1][c], qv[QW / 2][i], cv[CW / 2][c]))
          } else if (mode == SC_MODE_T) {
            KGE_FOR_PAIRS(acc_elem_mode<EL>(acc[i][c], SC_MODE_T, qv[0][i], qv[QW - 1][i], cv[0][c], cv[CW - 1][c], qv[QW / 2][i], cv[CW / 2][c]))
          } else {
            KGE_FOR_PAIRS(acc_elem_mode<EL>(acc[i][c], SC_MODE_T_FMA, qv[0][i], qv[QW - 1][i], cv[0][c], cv[CW - 1][c], qv[QW / 2][i], cv[CW / 2][c]))
          }
          if constexpr (CASC) {
            if (code & SC_CASC1) { KGE_FOR_PAIRS(acc_casc1(acc[i][c])) }
            if (code & SC_FOLD1) { KGE_FOR_PAIRS(acc_fold1(acc[i][c])) }
          }
          if (code & SC_P_SET) { KGE_FOR_PAIRS(acc_p_set(acc[i][c])) }
          if (code & SC_P_ADD) { KGE_FOR_PAIRS(acc_p_add(acc[i][c])) }
          if (code & SC_T_ADD_P) { KGE_FOR_PAIRS(acc_t_add_p(acc[i][c])) }
          if (code & SC_T_ADD_A) { KGE_FOR_PAIRS(acc_t_add_a(acc[i][c])) }
        }
      };
      if constexpr (APPROX) {
#pragma unroll 4
        for (int kk = 0; kk < kn; ++kk) {
          float qv[QW][TQ], cv[CW][TC];
          load_operands(kk, qv, cv);
          KGE_FOR_PAIRS(acc[i][c].a += elem_rot_fast(qv[0][i], qv[QW - 1][i], cv[0][c], cv[CW - 1][c]))
        }
        KGE_FOR_PAIRS(acc[i][c].t += acc[i][c].a; acc[i][c].a = 0.f)
      } else {
        // run-length form: branch-free unrolled runs of ordinary positions between flagged ones
        uint32_t m = special;
        int kk = 0;
        while (kk < kn) {
          const int run = m ? min(kn - kk, __ffs(m) - 1) : kn - kk;
#pragma unroll 4
          for (int j = 0; j < run; ++j) {
            float qv[QW][TQ], cv[CW][TC];
            load_operands(kk + j, qv, cv);
            KGE_FOR_PAIRS(acc_step_fast<EL>(acc[i][c], qv[0][i], qv[QW - 1][i], cv[0][c], cv[CW - 1][c], qv[QW / 2][i], cv[CW / 2][c]))
          }
          kk += run;
          if (kk < kn) {
            float qv[QW][TQ], cv[CW][TC];
            load_operands(kk, qv, cv);
            consume(kk, qv, cv);  // flagged by construction
            ++kk;
            m = (run + 1 >= 32) ? 0u : (m >> (run + 1));
          }
        }
      }
#undef KGE_FOR_PAIRS
      __syncwarp();
      if (lane == 0) ptx::mbar_arrive(&empty_bar[stage]);
      if (++stage == STAGES) { stage = 0; phase ^= 1u; }
    }

    // ---- epilogue: finish the scores, count or store ----
    const long long c_base = ct * TILE_C + c_off;
    if (p.col_buf != nullptr) {
      // top-k collect: keep what is not below the query's current k-th best (NaN kept: torch.topk
      // ranks NaN above everything)
#pragma unroll
      for (int i = 0; i < TQ; ++i) {
        const long long q = qt * TILE_Q + q_off + i;
        if (q >= p.n_q) continue;
        int2* list = p.col_buf + (size_t)q * p.col_cap;
#pragma unroll
        for (int j = 0; j < TC; ++j) {
          const long long c = c_base + 32 * (j / 4) + (j % 4);
          if (c >= p.n_rows) continue;
          const float s = acc_finish<EL>(acc[i][j]);
          if (!(s < st[i])) {
            const unsigned long long slot = p.col_dense ? (unsigned long long)c
                                                        : (unsigned long long)atomicAdd(&p.col_count[q], 1u);
            if (slot < p.col_cap) list[slot] = make_int2(__float_as_int(s), (int)(p.col_id_base + c));
          }
        }
      }
    } else if (p.scores != nullptr) {
#pragma unroll
      for (int i = 0; i < TQ; ++i) {
        const long long q = qt * TILE_Q + q_off + i;
        if (q >= p.n_q) continue;
        float* row = p.scores + (size_t)q * p.n_rows;
#pragma unroll
        for (int j = 0; j < TC; ++j) {
          const long long c = c_base + 32 * (j / 4) + (j % 4);
          if (c < p.n_rows) row[c] = acc_finish<EL>(acc[i][j]);
        }
      }
    } else if constexpr (APPROX) {
      const bool edge = (ct * TILE_C + TILE_C > p.n_rows);
#pragma unroll
      for (int j = 0; j < TC; ++j) {
        const long long c = c_base + 32 * (j / 4) + (j % 4);
        const bool valid = !edge || (c < p.n_rows);
#pragma unroll
        for (int i = 0; i < TQ; ++i) {
          const float s = -acc[i][j].t;
          const bool gt = s > t_hi[i], lt = s < t_lo[i];
          cnt[i] += (valid && gt) ? 1 : 0;
          if (valid && !gt && !lt) {  // near-tie (or NaN): exact recheck decides
            const long long q = qt * TILE_Q + q_off + i;
            if (q < p.n_q) {
              const long long region = q / 128;
              const unsigned long long slot = atomicAdd(p.amb_count + region, 1ull);
              if (slot < p.amb_cap) p.amb_pairs[(size_t)region * p.amb_cap + slot] = make_int2((int)q, (int)c);
            }
          }
        }
      }
    } else {
      const bool edge = (ct * TILE_C + TILE_C > p.n_rows);
#pragma unroll
      for (int j = 0; j < TC; ++j) {
        const long long c = c_base + 32 * (j / 4) + (j % 4);
        const bool valid = !edge || (c < p.n_rows);
#pragma unroll
        for (int i = 0; i < TQ; ++i) {
          const float s = acc_finish<EL>(acc[i][j]);
          cnt[i] += (valid && s >= st[i]) ? 1 : 0;
        }
      }
    }
  }
  flush_counts(cur_qt);
}

template <int EL, bool CASC, int G, bool APPROX = false>
cudaError_t launch_one(ScanParams& p, cudaStream_t stream) {
  using L = Cfg<EL, G>;
  // stage masks: which positions are NOT the plain "accumulate" code of this reduction kind
  constexpr uint8_t FAST = ElemTraits<EL>::RED == RED_SEQ ? SC_MODE_T : SC_MODE_A;
  const int n_kc = (p.dim + KC - 1) / KC;
  for (int kc = 0; kc < n_kc; ++kc) {
    uint32_t m = 0;
    for (int kk = 0; kk < KC && kc * KC + kk < p.dim; ++kk)
      if (p.code[kc * KC + kk] != FAST) m |= 1u << kk;
    p.mask[kc] = m;
  }
  constexpr auto kern = scan_kernel<EL, CASC, G, APPROX>;
  cudaError_t e = set_attribute_once<kern>(cudaFuncAttributeMaxDynamicSharedMemorySize, (int)L::SMEM_BYTES);
  if (e != cudaSuccess) return e;
  int dev = 0, sms = 0;
  e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  if (e != cudaSuccess) return e;
  const long long total = (long long)p.n_qt * (long long)p.n_ct;
  if (total <= 0) return cudaSuccess;
  const int grid = (int)(total < sms ? total : sms);
  kern<<<grid, L::THREADS, L::SMEM_BYTES, stream>>>(p);
  return cudaGetLastError();
}

template <int G>
cudaError_t launch_scan_g(int el, bool cascade, ScanParams& p, cudaStream_t stream, bool approx) {
  if (approx) {
    if (el != EL_ROT || p.amb_count == nullptr || p.amb_pairs == nullptr || p.scores != nullptr)
      return cudaErrorInvalidValue;
    return cascade ? launch_one<EL_ROT, true, G, true>(p, stream) : launch_one<EL_ROT, false, G, true>(p, stream);
  }
  return dispatch_elem(el, cascade, [&](auto kind, auto casc) {
    return launch_one<decltype(kind)::value, decltype(casc)::value, G>(p, stream);
  });
}

}  // namespace

cudaError_t launch_scan(int el, bool cascade, const ScanParams& p_in, cudaStream_t stream, bool approx) {
  if (p_in.dim < 1 || p_in.dim > SCAN_MAX_DIM - 1 || p_in.code_host == nullptr)
    return cudaErrorInvalidValue;
  ScanParams p = p_in;
  memcpy(p.code, p_in.code_host, (size_t)p.dim);
  // Thread tile 4 x 4 pairs, 16 warps per CTA (G = 2 gives 4 x 8 / 8 warps).
  return launch_scan_g<1>(el, cascade, p, stream, approx);
}

}  // namespace kge
