// Tensor-core bound-and-refine path: shared definitions (tc.cu, api.cu).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <type_traits>

namespace kge {
namespace tc {

constexpr int TC_BM = 128;       // queries per MMA tile (two wgmma M = 64 halves)
constexpr int TC_BN = 256;       // candidates per MMA tile (wgmma N)
// k-block width (bf16 per swizzle span) is a run-time choice: bk() = 32 (64-byte swizzle,
// default) or 64 (128-byte swizzle, KGE_TC_BK=64); n_kblocks(k_total) = ceil(k_total / bk()).
int bk();
int n_kblocks(int k_total);
// Tuning / test hook (kge_tc_configure): bk 32|64, resident 0|1, ct_group (0 = automatic),
// max_ctas (0 = one per SM), fp16 0|1 (operand format of the split, see below); negative values
// keep the current setting.  Operand images packed under one (bk, fp16) must be scanned under the same.
void configure(int bk, int resident, int ct_group, int max_ctas, int fp16);
// Operand format of the split x = hi + lo: bf16 (8 significant bits each, residual 2^-16 |x|) or
// fp16 (11 bits each, residual 2^-22 |x|, operands pre-scaled by a power of two per table so that
// the lo parts stay in fp16's normal range; the default: the smaller residual narrows the near-tie
// band).  KGE_TC_FP16=0|1.
bool fp16();

// Per-operand facts the pack kernels establish ON THE DEVICE (no host round trip) and the scan
// reads: 32 bytes at the end of the candidate image (B) / in the call's workspace (A).
struct TcMeta {
  float scale;      // power of two the operand was multiplied by (1 for bf16); NaN: operand has non-finite
                    // entries or its range cannot be represented -> every pair goes to the exact recheck
  float max_abs;    // max |x| over the operand        (bit pattern maximum: NaN / inf win)
  float max_norm2;  // max row |x|^2
  float fold;       // B: phi (the fold slots hold -|b|^2/2 * phi);  A: alpha (its fold slots hold alpha)
  float acc_scale;  // A only: S = scale_a * scale_b = alpha * phi; the accumulator holds S * (a.b - |b|^2/2)
  float e_abs;      // A only: absolute error (score units) of the scaled representation
  float kappa;      // added to every row's norm bound (covers the absolute residual of subnormal lo parts)
  float reserved;
};
constexpr size_t TC_META_BYTES = 256;

struct TcScanParams {
  const unsigned char* apack = nullptr;  // [n_qt][n_kb][hi,lo][128 rows x 2*bk() B, swizzled]
  const unsigned char* bpack = nullptr;  // [n_ct][n_kb][hi,lo][256 rows x 2*bk() B, swizzled]
  const float* s_true = nullptr;         // [n_q] exact (ATen-order) true scores
  const float* qbound = nullptr;         // [n_q] >= |a|_2
  const float* qnorm2 = nullptr;         // [n_q] |a|_2^2 (L2 only)
  const float* cbound = nullptr;         // [n_rows] >= |b|_2
  const float* cnorm2 = nullptr;         // [n_rows]
  const float* qprefix = nullptr;        // [n_q]    P(a) = sqrt(sum_i |a_{<=16 i}|^2): running-magnitude factor (tc_gamma_p)
  const float* cprefix = nullptr;        // [n_rows] P(b)
  const float* cbmax32 = nullptr;        // [n_ct * 8] max of cbound over each aligned block of 32 rows
  const float* cpmax32 = nullptr;        // [n_ct * 8] max of cprefix over each aligned block of 32 rows
  int32_t* counts = nullptr;             // [n_q] +=
  unsigned long long* amb_count = nullptr;  // [n_qt] fill count of each query tile's region
  int2* amb_pairs = nullptr;                // [n_qt][amb_cap]
  unsigned long long amb_cap = 0;           // capacity of ONE region
  float* dump = nullptr;                 // debug: write approximate scores [n_q][n_rows] instead of counting
  const TcMeta* meta_a = nullptr;        // device: facts of the query image (this call)
  const TcMeta* meta_b = nullptr;        // device: facts of the candidate image
  int fp16 = 0;                          // operand format of the images: 1 = fp16, 0 = bf16 (set by launch_tc_scan)
  float gamma = 0.f;                     // tc_gamma(k): multiplies |a| |b|
  float gamma2 = 0.f;                    // tc_gamma2(k) (L2 only): multiplies (|a| + |b|)^2
  float gamma_p = 0.f;                   // tc_gamma_p(): multiplies P(a) P(b) (accumulation inside the tensor core)
  int l2 = 0;                            // 1: score = -(|a|^2 + |b|^2 - 2 a.b)
  int n_kb = 0;
  int k_total = 0;
  int ct_group = 0;                      // candidate tiles a CTA walks per query tile (set by launch_tc_scan)
  long long n_q = 0, n_rows = 0, n_qt = 0, n_ct = 0;
};
static_assert(std::is_trivially_copyable<TcScanParams>::value, "TcScanParams is a kernel parameter");

// Rigorous bound eps >= |s_tc - s_ATen| used by the threshold test:
//   dot models : eps = gamma  * |a| |b|
//   L2         : eps = gamma  * 2 |a| |b|  +  gamma2 * (|a| + |b|)^2
// gamma collects everything proportional to sum_k |a_k b_k| <= |a| |b|:
//   splitting x = hi + lo + r into two half-precision numbers (two roundings to p significant bits:
//     p = 8 for bf16, 11 for fp16), |r| <= 2^-2p |x|; dropped lo*lo, a*r_b, r_a*b
//                                                                   -> 3 * 2^-2p (1 + 2^-p)  (exact bound)
//     (fp16 only: a lo part below fp16's normal range is off by <= 2^-25 in scaled units instead;
//      that absolute residual is carried by TcMeta::kappa, an additive inflation of the row bounds)
//   fp32 accumulation inside the tensor core: every wgmma k-step adds 16 exact products to the
//     accumulator; MEASURED on an H100 SXM (scripts/tc_numerics_probe.py, tests/golden/tc_numerics_probe*.json):
//     |result - exact| <= TC_ACC_ULPS * 2^-24 * (|acc_in| + sum |products|) per instruction.
//     Summed over the 3 ceil(k/16) instructions of a pair: the products are counted once,
//     sum |products| <= (1 + 2^-p)^2 sum_k |a_k b_k|                      -> 1.01 TC_ACC_ULPS 2^-24  (in gamma)
//     and the incoming accumulator of any of the three instructions of k-step i is at most the sum
//     of the |products| of the first i k-steps, <= 1.01 |a_{<=16 i}| |b_{<=16 i}| (Cauchy-Schwarz on the
//     prefix), so that, with P(x)^2 = sum_i |x_{<=16 i}|^2 (per row, row_norms_kernel),
//       sum over instructions of |acc_in| <= 3.03 sum_i |a_{<=16i}| |b_{<=16i}| <= 3.03 P(a) P(b)
//                                                     -> gamma_p = 3.04 TC_ACC_ULPS 2^-24, times P(a) P(b)
//     (P(x) <= sqrt(ceil(k/16)) |x|: never worse than charging every instruction the full |a| |b|, and
//      about half of that when the mass of the vectors is spread evenly over k)
//   dot models only: the reference's own fp32 evaluation -- every product rounded once (ComplEx:
//     two products and their sum), then summed in ATen's cascade order, whose tree depth
//     `ref_depth` (schedule.h: schedule_depth, computed from the very schedule the exact kernels
//     replay) gives |fl(sum) - sum| <= ref_depth * u * sum|terms|   -> (ref_depth + 4) * 2^-24
// gamma2 (L2 only) collects what is proportional to the squared norms, (|a| + |b|)^2 >= |a - b|^2:
//   the reference forms x_k = q_k - c_k (head side: (c_k + r_k) - t_k, two roundings, |x| bounded
//   by |c| + |r| + |t| -- the head-side query bound is |t| + |r| for that reason), squares it,
//   sums in the 8-lane norm order (depth ref_depth), takes an exactly rounded sqrt and squares it:
//     relative (ref_depth + 10) u on sum x^2;
//   this side: |a|^2 and |b|^2 rounded to fp32 (2u), |b|^2/2 carried as three half-precision pieces
//   (u), the <= 6 MMA instructions that see it in their accumulator (6 TC_ACC_ULPS u |b|^2 / 2), threshold
//   arithmetic is directed-rounded                     -> (ref_depth + 18 + 3 TC_ACC_ULPS) * 2^-24
// tests/test_tc_gpu.py measures the actual error on random AND adversarial operands (cancelling,
// wide dynamic range, same sign) and requires error <= bound.
// What scripts/tc_numerics_probe.py found on an H100 SXM (tests/golden/tc_numerics_probe*.json): one
// wgmma k-step (bf16 or fp16 operands, f32 accumulator) aligns its 17 addends -- the incoming
// accumulator and the 16 exact products -- to the
// largest exponent among them, keeps each down to 2^-25 of that exponent (two bits below the fp32
// ulp; lower bits are cut toward zero: 1 + 15 x 2^-25 gives 1 + 3 ulp, 1 + 15 x 2^-26 gives 1), adds
// exactly and cuts the sum toward zero to 24 bits.  Hence per instruction
//   |result - exact| < 16 * 2^-25 * 2^Emax + 2^-23 |result| <= (8 + 2) * 2^-24 * (|acc_in| + sum |products|)
// Largest value observed on random operands (H100): 4.3 with bf16, 5.1 with fp16 operands (same-sign,
// wide exponent range).
// tests/test_tc_model_cpu.py replays this model in exact arithmetic against every crafted probe result.
constexpr double TC_ACC_ULPS = 10.0;  // per-instruction accumulation error in units of 2^-24 * running magnitude
inline float tc_gamma(int k_total, int ref_depth, bool l2, bool fp16 = false) {
  const double split = fp16 ? 3.0 * 0x1p-22 * (1.0 + 0x1p-11) : 3.0 * 0x1p-16 * (1.0 + 0x1p-8);
  const double accum_once = 1.01 * TC_ACC_ULPS * 0x1p-24;   // the products themselves, counted once
  const double ref = l2 ? 0.0 : (ref_depth + 4.0) * 0x1p-24;
  (void)k_total;
  return (float)(split + accum_once + ref);
}
inline float tc_gamma_p() { return (float)(3.04 * TC_ACC_ULPS * 0x1p-24); }
inline float tc_gamma2(int ref_depth) { return (float)((ref_depth + 18.0 + 3.0 * TC_ACC_ULPS) * 0x1p-24); }

size_t a_image_bytes(long long n_q, int n_kb);
size_t b_image_bytes(long long n_rows, int n_kb);
// fold = true (L2 models, k_total = dim + 3): the images carry -|b|^2/2 resp. 1.0 in the three k
// slots after the data, so the accumulator already holds  a.b - |b|^2/2.
// meta_b / meta_a: TC_META_BYTES of device memory each (written here, read by the scan).
// guard (launch_pack_b, optional): 4 device uint64 kept by the caller NEXT TO a cached image: the
// table's content checksum is recomputed (one read of the table) and the packing kernels run only
// if it differs from the checksum the image was built from -- a cache that cannot go stale.
cudaError_t launch_pack_b(const float* ent0, const float* ent1, long long n_rows, int dim, int k_total,
                          int n_kb, bool fold, unsigned char* bpack, float* cbound, float* cnorm2, float* cprefix,
                          float* cbmax32, float* cpmax32, TcMeta* meta_b, unsigned long long* guard, cudaStream_t st);
cudaError_t launch_pack_a(const float* qplain, int qw, long long n_q, int dim, int k_total, int n_kb,
                          int sub_mode, bool fold, unsigned char* apack, float* qbound, float* qnorm2, float* qprefix,
                          TcMeta* meta_a, const TcMeta* meta_b, cudaStream_t st);
cudaError_t launch_tc_scan(const TcScanParams& p, cudaStream_t st);
// The near-tie list is split into one region per QUERY TILE (regions = n_qt): region_counts[regions]
// (zeroed by the caller), pairs[regions][region_cap].  A region's pairs all belong to the same 128
// queries, whose rows therefore stay L1-resident during the exact recheck of that region.
int scan_grid_size(long long n_q, long long n_rows, int n_kb, int* group_out = nullptr);
cudaError_t launch_recheck(int el, int dim, const unsigned long long* region_counts, int regions,
                           unsigned long long region_cap, const int2* pairs, const float* qplain,
                           const float* ent0, const float* ent1, const float* s_true, int32_t* counts,
                           unsigned long long* stats, cudaStream_t st);

}  // namespace tc
}  // namespace kge
