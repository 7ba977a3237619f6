// Tensor-core bound-and-refine for the rank scan (wgmma, sm_90a).
//
// For the models whose score is a dot product or a squared L2 distance (DistMult, RESCAL,
// ComplEx, TransE-L2) the count  #{c : s(q,c) >= s_true(q)}  does not need every score to the
// last bit: it needs every score to be on the right SIDE of s_true.  This kernel computes an
// approximation s~(q,c) on the tensor cores -- fp32 operands split into half-precision (hi, lo)
// pairs, three products per term (hi*hi + lo*hi + hi*lo), fp32 accumulation in registers --
// together with a rigorous bound eps(q,c) >= |s~ - s_ATen| (tc.h).  Pairs with
// |s~ - s_true| > eps are decided from s~; the few others (the "near-tie band") are appended to a
// list and re-scored exactly, with the ATen-order arithmetic, by recheck_kernel.  Ranks therefore
// stay bit-identical to the reference's while almost all of the arithmetic moves from the fp32
// pipes to the tensor cores.
//
// Kernel shape: persistent CTAs of 9 warps, one per SM.  Warp 8 (one lane): producer -- 1-D bulk
// async copies of pre-swizzled operand images (the pack kernels write the exact shared-memory
// image of K-major swizzled tiles, so no tensor map is needed): k-blocks of 32 half-precision
// values (64-byte swizzle) with the query tile's image resident for a whole work unit and the
// candidate image streaming through a 3-stage ring, or both streamed (4 x 48 KB; 2 x 96 KB with
// 128-byte swizzle).  Warps 0-7: two consumer warpgroups.  Warpgroup g issues wgmma
// (M=64 query rows 64g..64g+63 of the tile x N=256 candidates x K=16, -> f32 in registers) and
// then runs the epilogue on its own accumulator: compare with two per-row thresholds, count,
// append near-ties.
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <stdlib.h>

#include "kernels.h"
#include "ptx.cuh"
#include "tc.h"

namespace kge {
namespace tc {

namespace {

constexpr int BM = TC_BM, BN = TC_BN;
constexpr int AMB_BUF = 64;          // near-tie entries buffered per consumer warp
constexpr int MMA_WARPS = 8;         // two warpgroups, 64 query rows each
constexpr int PRODUCER_WARP = MMA_WARPS;   // first warp of the third warpgroup
constexpr int THREADS = (MMA_WARPS + 4) * 32;
// registers per thread after the hand-over (setmaxnreg): 128 x 40 + 256 x 232 <= 64 K
constexpr int PRODUCER_REGS = 40, CONSUMER_REGS = 232;
constexpr int ACC = BN / 2;          // fp32 accumulator registers per thread (m64n256)
constexpr int MAX_STAGES = 4;
constexpr int BAR_SLOTS = 32;        // full[4] empty[4] a_full[8] a_empty[1] ...
constexpr int BLOCKS = TC_BN / 32;   // 32-column blocks of a candidate tile
// barriers, near-tie buffers, and (T_hi, T_lo) of both rows of each lane quad for each block
constexpr size_t SMEM_TAIL = BAR_SLOTS * sizeof(uint64_t) + MMA_WARPS * AMB_BUF * sizeof(int2) +
                             MMA_WARPS * BLOCKS * 8 * sizeof(float4);
constexpr size_t SMEM_LIMIT = 232448;  // 227 KB opt-in maximum per CTA on sm_90

// Geometry of one kernel variant: BKT half-precision values per k-block (= one swizzle span of
// 2*BKT bytes); RES = the query tile's whole A image stays resident in shared memory for a unit
// and only B is streamed (possible when the image is <= 7 k-blocks of 32, i.e. k_total <= 224).
template <int BKT, bool RES>
struct Geo {
  static constexpr int ROWB = 2 * BKT;                 // bytes per operand row in a k-block
  static constexpr int A_PLANE = BM * ROWB;            // one 128-row (hi or lo) plane
  static constexpr int B_PLANE = BN * ROWB;
  static constexpr int A_BLOCK = 2 * A_PLANE;          // hi + lo
  static constexpr int B_BLOCK = 2 * B_PLANE;
  static constexpr int STAGE_BYTES = RES ? B_BLOCK : A_BLOCK + B_BLOCK;
  static constexpr int STAGES = RES ? 3 : (BKT == 64 ? 2 : 4);
  static constexpr int K16 = BKT / 16;                 // MMA k-steps per block
  static constexpr uint64_t LAYOUT = BKT == 64 ? 1 : 2;  // wgmma descriptor: SWIZZLE_128B : SWIZZLE_64B
  static constexpr uint32_t SBO = 8 * ROWB;            // byte stride between 8-row groups
};

template <int BKT, bool RES>
size_t smem_bytes(int n_kb) {
  using G = Geo<BKT, RES>;
  return 1024 /*align slack*/ + (RES ? (size_t)n_kb * G::A_BLOCK : 0) + (size_t)G::STAGES * G::STAGE_BYTES +
         SMEM_TAIL;
}

// -------- wgmma helpers --------
// K-major swizzled shared-memory matrix descriptor: start address >> 4 | LBO = 1 (unused for
// swizzled K-major) | SBO = 8 rows x row bytes | layout type in bits [62,64) (1 = SWIZZLE_128B for
// 128-byte rows, 2 = SWIZZLE_64B for 64-byte rows).  Advancing K by 16 values inside the swizzle
// span adds 32 bytes (2 units of 16) to the start address.
template <class G>
__device__ __forceinline__ uint64_t make_desc(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)(G::SBO >> 4) << 32;
  d |= G::LAYOUT << 62;
  return d;
}
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator accesses across the asynchronous MMAs
__device__ __forceinline__ void fence_acc(float (&d)[ACC]) {
#pragma unroll
  for (int i = 0; i < ACC; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// D[regs] (+)= A[smem] * B[smem]^T, 64 x 256 x 16, both operands K-major; accumulate = 0 overwrites D.
// Accumulator layout (thread t of the warpgroup, warp w = t / 32, lane l): d[i] is row
// 16 w + l / 4 + 8 ((i >> 1) & 1), column 8 (i >> 2) + 2 (l & 3) + (i & 1).
template <bool FP16>
__device__ __forceinline__ void wgmma(float (&d)[128], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
// AB: the operand types of the instruction, the only part that depends on the format
#define KGE_WGMMA(AB)                                                                                                   \
  asm volatile(                                                                                                         \
      "{\n\t"                                                                                                           \
      ".reg .pred p;\n\t"                                                                                               \
      "setp.ne.b32 p, %130, 0;\n\t"                                                                                     \
      "wgmma.mma_async.sync.aligned.m64n256k16.f32." AB " "                                                             \
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "                                         \
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "                                \
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "                                \
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "                                \
      "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, "                                \
      "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, "                                \
      "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, "                    \
      "%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, "               \
      "%128, %129, p, 1, 1, 0, 0;\n\t"                                                                                  \
      "}\n"                                                                                                             \
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),                 \
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),           \
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),         \
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),         \
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),         \
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),         \
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),         \
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),         \
        "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),         \
        "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),         \
        "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]),         \
        "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]),         \
        "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]),     \
        "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), \
        "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), \
        "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])  \
      : "l"(desc_a), "l"(desc_b), "r"(accumulate)                                                                       \
      : "memory")
  if constexpr (FP16) KGE_WGMMA("f16.f16");
  else KGE_WGMMA("bf16.bf16");
#undef KGE_WGMMA
}

// Threshold tests as one FSET each: the bits of 1.0f (0x3F800000) when the test passes, else 0.
// (ptxas lowers an integer-valued set to FSETP + SEL, two instructions.)  A sum of n such words is
// n * 127 * 2^23 (mod 2^32): equal sums mean equal counts for n < 512, and ones_count() recovers n.
// a > b (false when either is NaN)
__device__ __forceinline__ uint32_t one_if_gt(float a, float b) {
  float r;
  asm("set.gt.f32.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
  return __float_as_uint(r);
}
// a >= b or unordered (true when either is NaN)
__device__ __forceinline__ uint32_t one_if_geu(float a, float b) {
  float r;
  asm("set.geu.f32.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
  return __float_as_uint(r);
}
// n from the sum of n words 0x3F800000, n < 512: 127 is odd and 383 * 127 = 1 (mod 512)
__device__ __forceinline__ int ones_count(uint32_t sum) { return (int)(((sum >> 23) * 383u) & 511u); }


// Work order: a unit = (group of p.ct_group consecutive candidate tiles, query tile); a CTA
// takes units round-robin and walks the group's candidate tiles for that query tile.  CTAs
// running together work on the same group with different query tiles, so the group's B images
// are served from L2 (B streams from HBM once per launch) and the whole A image (tens of MB)
// stays L2-resident; per-query counters are flushed once per unit.
struct Units {
  long long n_qt, n_ct, grp, n_units;
  __device__ Units(long long nq, long long nc, long long g)
      : n_qt(nq), n_ct(nc), grp(g), n_units(nq * ((nc + g - 1) / g)) {}
  __device__ void decode(long long u, long long* qt, long long* ct_lo, long long* ct_hi) const {
    const long long g = u / n_qt;
    *qt = u - g * n_qt;
    *ct_lo = g * grp;
    *ct_hi = min(n_ct, *ct_lo + grp);
  }
};

// Appends this warp's near-ties of one 32-column block to its shared buffer (flushed to the query
// tile's region of the global list when full); bit e of `mask` is accumulator element 16 b + e.
struct NearTies {
  int2* wbuf;
  int amb_n;                 // entries in wbuf (warp-uniform)
  __device__ void flush(const TcScanParams& p, long long qt, int lane) {
    __syncwarp();
    unsigned long long base = 0;
    if (lane == 0) base = atomicAdd(p.amb_count + qt, (unsigned long long)amb_n);
    base = __shfl_sync(0xffffffffu, base, 0);
    for (int i = lane; i < amb_n; i += 32)
      if (base + i < p.amb_cap) p.amb_pairs[(size_t)qt * p.amb_cap + base + i] = wbuf[i];
    __syncwarp();
    amb_n = 0;
  }
  __device__ void append(const TcScanParams& p, long long qt, int lane, unsigned mask, long long q0, long long c0) {
    // q0: query of the thread's first row (the second is q0 + 8); c0: column of element 0
    const int mine = __popc(mask);
    int incl = mine;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int up = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += up;
    }
    const int total_new = __shfl_sync(0xffffffffu, incl, 31);
    auto entry = [&](int e) {
      return make_int2((int)(q0 + 8 * ((e >> 1) & 1)), (int)(c0 + 8 * (e >> 2) + (e & 1)));
    };
    if (amb_n + total_new > AMB_BUF) flush(p, qt, lane);   // uniform decision
    if (total_new <= AMB_BUF) {
      int slot = amb_n + incl - mine;
      unsigned m = mask;
      while (m) {
        const int e = __ffs(m) - 1;
        m &= m - 1;
        wbuf[slot++] = entry(e);
      }
      amb_n += total_new;
    } else {
      // pathological block (more near-ties than the buffer holds): straight to global
      unsigned long long base = 0;
      if (lane == 0) base = atomicAdd(p.amb_count + qt, (unsigned long long)total_new);
      base = __shfl_sync(0xffffffffu, base, 0) + (unsigned long long)(incl - mine);
      unsigned m = mask;
      while (m) {
        const int e = __ffs(m) - 1;
        m &= m - 1;
        if (base < p.amb_cap) p.amb_pairs[(size_t)qt * p.amb_cap + base] = entry(e);
        ++base;
      }
    }
  }
};

template <bool L2, bool DUMP, bool FP16, int BKT, bool RES>
__global__ void __launch_bounds__(THREADS, 1) tc_scan_kernel(const __grid_constant__ TcScanParams p) {
  using G = Geo<BKT, RES>;
  constexpr int STAGES = G::STAGES;
  extern __shared__ unsigned char smem_raw[];
  // 1024-B alignment for the swizzle atoms
  const uint32_t raw_addr = ptx::smem_u32(smem_raw);
  unsigned char* smem = smem_raw + ((1024 - (raw_addr & 1023)) & 1023);
  const int n_kb = p.n_kb;
  unsigned char* a_res = smem;  // [n_kb][hi, lo][128 rows]   (RES only)
  unsigned char* stage_base = smem + (RES ? (size_t)n_kb * G::A_BLOCK : 0);
  uint64_t* bars = reinterpret_cast<uint64_t*>(stage_base + (size_t)STAGES * G::STAGE_BYTES);
  uint64_t* full_bar = bars;             // [MAX_STAGES]
  uint64_t* empty_bar = bars + 4;        // [MAX_STAGES]  one arrival per consumer warp
  uint64_t* afull_bar = bars + 8;        // [8]  one per resident A k-block
  uint64_t* aempty_bar = bars + 16;      // [1]  resident A region free again (one arrival per consumer warp)
  int2* s_amb = reinterpret_cast<int2*>(bars + BAR_SLOTS);  // [MMA_WARPS][AMB_BUF]
  float4* s_thr = reinterpret_cast<float4*>(s_amb + MMA_WARPS * AMB_BUF);   // [MMA_WARPS][BLOCKS][8 quads]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const Units units(p.n_qt, p.n_ct, p.ct_group);

  if (threadIdx.x == 0) {
    for (int s = 0; s < MAX_STAGES; ++s) {
      ptx::mbar_init(&full_bar[s], 1);
      ptx::mbar_init(&empty_bar[s], MMA_WARPS);
    }
    for (int k = 0; k < 8; ++k) ptx::mbar_init(&afull_bar[k], 1);
    ptx::mbar_init(aempty_bar, MMA_WARPS);
    ptx::fence_mbar_init();
  }
  __syncthreads();

  if (warp >= PRODUCER_WARP) {
    // ------------------------------ producer ------------------------------
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(PRODUCER_REGS));
    if (warp == PRODUCER_WARP && lane == 0) {
      int stage = 0; uint32_t phase = 0;
      uint32_t unit_no = 0;
      for (long long u = blockIdx.x; u < units.n_units; u += gridDim.x, ++unit_no) {
        long long qt, ct_lo, ct_hi; units.decode(u, &qt, &ct_lo, &ct_hi);
        const unsigned char* asrc = p.apack + (size_t)qt * n_kb * G::A_BLOCK;
        if constexpr (RES) {
          // the previous unit's MMAs must have finished reading the resident A image
          if (unit_no > 0) ptx::mbar_wait(aempty_bar, (unit_no - 1) & 1u);
          for (int kb = 0; kb < n_kb; ++kb) {
            ptx::mbar_arrive_expect_tx(&afull_bar[kb], G::A_BLOCK);
            ptx::bulk_g2s(a_res + (size_t)kb * G::A_BLOCK, asrc + (size_t)kb * G::A_BLOCK, G::A_BLOCK,
                          &afull_bar[kb]);
          }
        }
        for (long long ct = ct_lo; ct < ct_hi; ++ct) {
          const unsigned char* bsrc = p.bpack + (size_t)ct * n_kb * G::B_BLOCK;
          for (int kb = 0; kb < n_kb; ++kb) {
            ptx::mbar_wait(&empty_bar[stage], phase ^ 1u);
            unsigned char* sa = stage_base + (size_t)stage * G::STAGE_BYTES;
            ptx::mbar_arrive_expect_tx(&full_bar[stage], G::STAGE_BYTES);
            if constexpr (!RES) {
              ptx::bulk_g2s(sa, asrc + (size_t)kb * G::A_BLOCK, G::A_BLOCK, &full_bar[stage]);
              sa += G::A_BLOCK;
            }
            ptx::bulk_g2s(sa, bsrc + (size_t)kb * G::B_BLOCK, G::B_BLOCK, &full_bar[stage]);
            if (++stage == STAGES) { stage = 0; phase ^= 1u; }
          }
        }
      }
    }
    return;
  }

  // ------------------------------ consumers (warps 0..7) ------------------------------
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(CONSUMER_REGS));
  // The accumulator holds  f = a.b  (dot models) or  f = a.b - |b|^2/2  (L2: the candidate's
  // squared norm rides in three spare k slots of the operand images, see pack_operand_kernel),
  // so a pair is decided by comparing f with two per-row thresholds -- no per-candidate
  // loads, no arithmetic per element:
  //   dot: s~ = f,            u = s~ - s_true = f - st
  //   L2 : s~ = 2 f - |a|^2,  u = 2 f - (qn + st)
  //   eps(q, c) <= E(q, cbmax) with cbmax = max bound of the 32 candidates of the block
  //   (eps is increasing in the candidate's norm bound), hence
  //   f >  T_hi = (st + E)            [L2: (qn + st + E) / 2]  =>  s(q,c) >  s_true : count
  //   f <  T_lo = (st - E)            [L2: (qn + st - E) / 2]  =>  s(q,c) <  s_true : skip
  //   otherwise (including any NaN) near-tie: exact recheck.  T_hi is rounded up, T_lo down.
  const int wg = warp >> 2;                                     // warpgroup: tile rows 64 wg ..
  const int row0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);     // this thread's rows: row0, row0 + 8
  const int cq = 2 * (lane & 3);                                // its column offset in each 8-column chunk
  const uint32_t a_off = (uint32_t)(wg * 64 * G::ROWB);         // the warpgroup's 64 rows of an A plane
  int stage = 0; uint32_t phase = 0;
  uint32_t unit_no = 0;
  long long cur_qt = -1;
  float st[2] = {0.f, 0.f}, qn[2] = {0.f, 0.f}, kp[2] = {0.f, 0.f};
  float k1[2] = {0.f, 0.f}, k0[2] = {0.f, 0.f}, tbase[2] = {0.f, 0.f};
  int cnt[2] = {0, 0};
  NearTies amb{s_amb + warp * AMB_BUF, 0};
  float4* const thr = s_thr + warp * BLOCKS * 8 + (lane >> 2);   // [b * 8]: this quad's block b
  constexpr float INFL = 1.f + 0x1p-19f;      // covers the fp32 rounding of E's evaluation
  // the accumulator holds S * (a.b [- |b|^2/2]), S = scale_a * scale_b (a power of two; NaN when an
  // operand could not be represented: both threshold tests then fail and every pair is rechecked)
  const float S = p.meta_a->acc_scale;
  const float inv_S = 1.f / S;
  const float e_abs = p.meta_a->e_abs;
  const float kappa_a = p.meta_a->kappa, kappa_b = p.meta_b->kappa;
  float acc[ACC];
#pragma unroll
  for (int i = 0; i < ACC; ++i) acc[i] = 0.f;

  // Flushes what this warp holds for query tile qt: the rows' counts, then the near-tie buffer.  The
  // near-tie list is kept per QUERY TILE (region = qt) so that the exact recheck of a region touches
  // only that tile's 128 query rows (they stay L1-resident there).
  auto flush_tile = [&](long long qt) {
    if (qt < 0) return;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const long long pq = qt * BM + row0 + 8 * h;
      if (cnt[h] != 0 && pq < p.n_q) atomicAdd(&p.counts[pq], cnt[h]);
    }
    if (amb.amb_n > 0) amb.flush(p, qt, lane);
  };

  for (long long u = blockIdx.x; u < units.n_units; u += gridDim.x, ++unit_no) {
   long long qt, ct_lo, ct_hi; units.decode(u, &qt, &ct_lo, &ct_hi);
   for (long long ct = ct_lo; ct < ct_hi; ++ct) {
    const long long q0 = qt * BM + row0;
    if (qt != cur_qt) {
      flush_tile(cur_qt);
      cur_qt = qt;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const long long q = q0 + 8 * h;
        const bool vq = q < p.n_q;
        cnt[h] = 0;
        st[h] = vq ? p.s_true[q] : INFINITY;
        const float qb = vq ? __fadd_ru(p.qbound[q], kappa_a) : 0.f;
        qn[h] = vq ? p.qnorm2[q] : 0.f;
        // accumulation term: gamma_p P(a) P(b) (x2 for L2, whose score is 2 f - |a|^2)
        kp[h] = vq ? (L2 ? 2.f : 1.f) * p.gamma_p * p.qprefix[q] * INFL : 0.f;
        if constexpr (L2) {
          // E = 2 gamma qb cb + gamma2 (qb + cb)^2 = cb (k1 + gamma2 cb) + k0
          k1[h] = 2.f * (p.gamma + p.gamma2) * qb * INFL;
          k0[h] = p.gamma2 * qb * qb * INFL;
          tbase[h] = qn[h] + st[h];
        } else {
          k1[h] = p.gamma * qb * INFL;   // E = gamma qb cb
          tbase[h] = st[h];
        }
      }
    }
    const int ncols = (int)min((long long)BN, p.n_rows - ct * BN);
    // ---- MMAs: one commit group per k-block, the previous block's stage released once its group is done
    int prev = -1;
    fence_acc(acc);
    for (int kb = 0; kb < n_kb; ++kb) {
      if constexpr (RES) {
        if (ct == ct_lo) ptx::mbar_wait(&afull_bar[kb], unit_no & 1u);
      }
      ptx::mbar_wait(&full_bar[stage], phase);
      const uint32_t sb = ptx::smem_u32(stage_base + (size_t)stage * G::STAGE_BYTES);
      const uint32_t sa = (RES ? ptx::smem_u32(a_res + (size_t)kb * G::A_BLOCK) : sb) + a_off;
      const uint32_t sbb = RES ? sb : sb + G::A_BLOCK;
      const uint64_t a_hi = make_desc<G>(sa), a_lo = make_desc<G>(sa + G::A_PLANE);
      const uint64_t b_hi = make_desc<G>(sbb), b_lo = make_desc<G>(sbb + G::B_PLANE);
      const int k16s = min(G::K16, (p.k_total - kb * BKT + 15) / 16);
      wg_fence();
#pragma unroll
      for (int k = 0; k < G::K16; ++k) {
        if (k < k16s) {
          const uint64_t adv = (uint64_t)(k * 2);  // 16 values = 32 B = 2 x 16-B units
          wgmma<FP16>(acc, a_hi + adv, b_hi + adv, (kb | k) ? 1u : 0u);
          wgmma<FP16>(acc, a_lo + adv, b_hi + adv, 1u);
          wgmma<FP16>(acc, a_hi + adv, b_lo + adv, 1u);
        }
      }
      wg_commit();
      if constexpr (!DUMP) {
        if (kb == 0) {
          // The tile's thresholds, while the tensor cores run the first k-block: the four lanes
          // that share two query rows split the 8 column blocks, 2 each, and leave (T_hi, T_lo) of
          // both rows in shared memory for the epilogue.
          __syncwarp();   // the previous tile's epilogue has read its thresholds
#pragma unroll
          for (int i = 0; i < 2; ++i) {
            const int b = 2 * (lane & 3) + i;
            if (32 * b < ncols) {
              // largest candidate norm bound / running-magnitude factor of the block's 32
              // candidates (maxima over aligned blocks of 32 rows, precomputed with the image)
              const long long blk = (ct * BN) / 32 + b;
              const float cb = __fadd_ru(__ldg(p.cbmax32 + blk), kappa_b), cpm = __ldg(p.cpmax32 + blk);
              float t[4];
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                float e;
                if constexpr (L2) e = fmaf(cb, fmaf(p.gamma2 * INFL, cb, k1[h]), k0[h]) * INFL;
                else e = k1[h] * cb;
                e = __fadd_ru(__fmaf_ru(kp[h], cpm, e), e_abs);
                float t_hi = __fadd_ru(tbase[h], e), t_lo = __fadd_rd(tbase[h], -e);
                if constexpr (L2) { t_hi = __fmul_ru(t_hi, 0.5f); t_lo = __fmul_rd(t_lo, 0.5f); }
                // exact (power of two) unless it overflows, then still on the safe side
                t[2 * h] = __fmul_ru(t_hi, S);
                t[2 * h + 1] = __fmul_rd(t_lo, S);
              }
              thr[b * 8] = make_float4(t[0], t[1], t[2], t[3]);
            }
          }
        }
      }
      wg_wait<1>();
      if (prev >= 0 && lane == 0) ptx::mbar_arrive(&empty_bar[prev]);
      prev = stage;
      if (++stage == STAGES) { stage = 0; phase ^= 1u; }
    }
    wg_wait<0>();
    fence_acc(acc);
    if (lane == 0) {
      ptx::mbar_arrive(&empty_bar[prev]);
      if constexpr (RES) {
        if (ct == ct_hi - 1) ptx::mbar_arrive(aempty_bar);   // every MMA of the unit has read A
      }
    }

    // ---- epilogue ----
    __syncwarp();   // this tile's thresholds are in shared memory
    uint32_t ones_gt[2] = {0u, 0u};   // per row: the hot path's "count" results of the tile (<= 64)
#pragma unroll
    for (int b = 0; b < BN / 32; ++b) {
      const int c0 = 32 * b;
      if (c0 >= ncols) break;
      float t_hi[2], t_lo[2];
      if constexpr (!DUMP) {
        const float4 t = thr[b * 8];
        t_hi[0] = t.x; t_lo[0] = t.y; t_hi[1] = t.z; t_lo[1] = t.w;
      }
      // Each of the thread's 16 values gets two tests: f > T_hi ("count") and f >= T_lo or
      // unordered ("not below"); a pair is a near-tie when it passes the second test only.  (A NaN
      // accumulator or threshold -- what a NaN or inf operand, norm bound or scale leads to -- fails
      // the first test and passes the second: it lands in the near-tie list, i.e. is adjudicated by
      // the exact arithmetic.)
      if constexpr (DUMP) {
#pragma unroll
        for (int e = 0; e < 16; ++e) {
          const float f = acc[16 * b + e];
          const int h = (e >> 1) & 1;
          const long long q = q0 + 8 * h;
          const int c = c0 + 8 * (e >> 2) + cq + (e & 1);
          if (c < ncols && q < p.n_q)
            p.dump[(size_t)q * p.n_rows + ct * BN + c] = L2 ? fmaf(2.f, f * inv_S, -qn[h]) : f * inv_S;
        }
      } else {
        // Hot path: no bit masks, only sums of the test results -- per row for "count", over both
        // rows for "not below".  T_hi >= T_lo whenever neither is NaN (directed rounding of
        // tbase +- e, e >= 0), and a NaN threshold makes one test uniform over the row, so a value
        // that passes "count" also passes "not below": the two sums differ exactly when the
        // thread has a near-tie in the block.
        uint32_t s_gt0 = 0u, s_gt1 = 0u, s_ge = 0u;
#pragma unroll
        for (int e = 0; e < 16; ++e) {
          const float f = acc[16 * b + e];
          const int h = (e >> 1) & 1;
          if (h == 0) s_gt0 += one_if_gt(f, t_hi[0]);
          else s_gt1 += one_if_gt(f, t_hi[1]);
          s_ge += one_if_geu(f, t_lo[h]);
        }
        ones_gt[0] += s_gt0;
        ones_gt[1] += s_gt1;
        const bool edge = c0 + 32 > ncols;   // columns past the table (last tile only)
        // Cold path (blocks with a near-tie, and partial blocks): the same tests as bit masks
        if (__any_sync(0xffffffffu, edge || s_ge != s_gt0 + s_gt1)) {
          unsigned lt_mask = 0, gt_mask = 0;
#pragma unroll
          for (int e = 0; e < 16; ++e) {
            const float f = acc[16 * b + e];
            const int h = (e >> 1) & 1;
            gt_mask |= (f > t_hi[h] ? 1u : 0u) << e;
            lt_mask |= (f < t_lo[h] ? 1u : 0u) << e;
          }
          unsigned amb_mask = ~(gt_mask | lt_mask) & 0xFFFFu;
          if (edge) {
            unsigned keep = 0u;
#pragma unroll
            for (int e = 0; e < 16; ++e)
              if (c0 + 8 * (e >> 2) + cq + (e & 1) < ncols) keep |= 1u << e;
            amb_mask &= keep;
            // the sums above also counted the columns past the table
            const unsigned past = gt_mask & ~keep;
            cnt[0] -= __popc(past & 0x3333u);
            cnt[1] -= __popc(past & 0xCCCCu);
          }
          // padding rows of the last query tile have no list entries (their thresholds are +inf,
          // but a non-finite candidate norm bound turns them into NaN, which fails both tests)
          if (q0 >= p.n_q) amb_mask &= 0xCCCCu;
          if (q0 + 8 >= p.n_q) amb_mask &= 0x3333u;
          amb.append(p, qt, lane, amb_mask, q0, ct * BN + c0 + cq);
        }
      }
    }
    cnt[0] += ones_count(ones_gt[0]);
    cnt[1] += ones_count(ones_gt[1]);
   }
  }
  flush_tile(cur_qt);
}

// ------------------------------------------------------------------------------------------
// Operand packing: fp32 rows -> (hi, lo) bf16 planes in the shared-memory image of K-major
// swizzled tiles.  One thread per (row, 16-byte chunk): 8 consecutive k of one plane.
//   128-byte rows (BKT = 64, SWIZZLE_128B): offset of (row r, chunk j) inside a plane =
//       (r/8)*1024 + (r%8)*128 + ((j ^ (r%8)) * 16)              j = 0..7
//   64-byte rows  (BKT = 32, SWIZZLE_64B) :
//       (r/8)*512  + (r%8)*64  + ((j ^ ((r>>1)&3)) * 16)         j = 0..3
// (the swizzle XORs address bits [4,7) with bits [7,10), resp. bits [4,6) with bits [7,9)).
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ float operand_value(const float* __restrict__ p0,
                                               const float* __restrict__ p1, int dim, int k,
                                               int k_total) {
  if (k >= k_total) return 0.f;
  if (k < dim) return p0[k];
  if (k < 2 * dim) return p1[k - dim];
  // third plane of a three-plane row (Analogy: k_total = 3 dim): the planes are equally spaced, both in
  // a query row ([3][dim], p1 = p0 + dim) and across the stacked candidate table (include/kge_b200.h)
  return (p1 + (p1 - p0))[k - 2 * dim];
}

// Half-precision formats of the split: bf16 (8 significant bits) or fp16 (11; operands pre-scaled)
// Optional content guard of a cached candidate image: guard[0..1] = checksum of the table as it is
// now, guard[2..3] = checksum of the table the image was built from (0, 0 before the first build is
// committed; a real checksum has bit 0 of word 1 set).  Equal => every pack kernel returns at once.
__device__ __forceinline__ bool guard_unchanged(const unsigned long long* __restrict__ guard) {
  return guard != nullptr && guard[0] == guard[2] && guard[1] == guard[3];
}

template <bool FP16> struct HalfT;
template <> struct HalfT<false> {
  using T = __nv_bfloat16;
  static __device__ __forceinline__ T from(float x) { return __float2bfloat16_rn(x); }
  static __device__ __forceinline__ float to(T h) { return __bfloat162float(h); }
};
template <> struct HalfT<true> {
  using T = __half;
  static __device__ __forceinline__ T from(float x) { return __float2half_rn(x); }
  static __device__ __forceinline__ float to(T h) { return __half2float(h); }
};

template <int ROWS, int BKT, bool FP16>
__global__ void pack_operand_kernel(const float* __restrict__ src0, const float* __restrict__ src1,
                                    long long row_stride, long long plane1_offset, long long n_rows,
                                    int dim, int k_total, int n_kb, int sub_mode, int fold,
                                    const float* __restrict__ norm2, const TcMeta* __restrict__ meta,
                                    const unsigned long long* __restrict__ guard,
                                    unsigned char* __restrict__ out) {
  if (guard_unchanged(guard)) return;   // the image already holds exactly this table
  // src0 + row*row_stride = first plane of the row; second plane at +plane1_offset (same row)
  // or in src1 (separate table).  sub_mode = 1: value = plane1[k] - plane0[k]  (t - r, L2 head)
  // Every value is multiplied by meta->scale (a power of two: exact) before it is split.
  // fold (L2 only; k_total = dim + 3): the three k slots after the data carry, on the candidate
  // side (fold = 2), -|b|^2/2 * phi split exactly into three half-precision pieces (hi plane; lo
  // plane 0) and, on the query side (fold = 1), alpha = scale_a * scale_b / phi -- so the hi*hi
  // product adds -S |b|^2/2 to every accumulator and the epilogue compares the accumulator with
  // thresholds directly.
  using H = HalfT<FP16>;
  using HT = typename H::T;
  constexpr int CH = BKT / 8;        // 16-byte chunks per row
  constexpr int ROWB = 2 * BKT;
  const long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long n_tiles = (n_rows + ROWS - 1) / ROWS;
  const long long total = n_tiles * n_kb * ROWS * CH;
  if (gid >= total) return;
  const float scale = meta->scale, fold_c = meta->fold;
  const int j = (int)(gid % CH);
  long long rest = gid / CH;
  const int r = (int)(rest % ROWS);
  rest /= ROWS;
  const int kb = (int)(rest % n_kb);
  const long long tile = rest / n_kb;
  const long long row = tile * ROWS + r;
  HT hi[8], lo[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    const int k = kb * BKT + j * 8 + e;
    float x = 0.f;
    if (row < n_rows) {
      if (fold && k >= dim) {
        if (k < dim + 3) {
          if (fold == 1) {
            hi[e] = H::from(fold_c);                 // alpha: a power of two inside the format's range
          } else {
            float rem = -0.5f * norm2[row] * fold_c;  // phi: a power of two (exact)
            HT piece = H::from(rem);
            for (int i = 0; i < k - dim; ++i) {
              rem -= H::to(piece);  // exact: piece holds the leading bits of rem
              piece = H::from(rem);
            }
            hi[e] = piece;
          }
          lo[e] = H::from(0.f);
          continue;
        }
      } else {
        const float* a = src0 + (size_t)row * row_stride;
        const float* b = src1 ? src1 + (size_t)row * row_stride : a + plane1_offset;
        if (sub_mode) x = k < dim ? __fsub_rn(b[k], a[k]) : 0.f;
        else x = operand_value(a, b, dim, k, k_total);
      }
    }
    x *= scale;
    const HT h = H::from(x);
    hi[e] = h;
    lo[e] = H::from(x - H::to(h));
  }
  const size_t plane = (size_t)ROWS * ROWB;
  const size_t base = ((size_t)tile * n_kb + kb) * (2 * plane);
  const int sw = BKT == 64 ? (r & 7) : ((r >> 1) & 3);
  const size_t off = (size_t)(r / 8) * (8 * ROWB) + (size_t)(r % 8) * ROWB + (size_t)((j ^ sw) * 16);
  *reinterpret_cast<uint4*>(out + base + off) = *reinterpret_cast<const uint4*>(hi);
  *reinterpret_cast<uint4*>(out + base + plane + off) = *reinterpret_cast<const uint4*>(lo);
}

// per-row |x|_2 (rounded up a little), |x|_2^2 and the running-magnitude factor
//   P(x) = sqrt( sum_{i=1..ceil(k/16)} |x_{<= 16 i}|^2 )     (tc.h: tc_gamma_p)
// of the operand vector, one warp per row: 32 consecutive k per iteration, lanes 0-15 / 16-31 are the
// two MMA k-steps of the iteration.  The operand's largest |x| and largest |x|_2^2 are folded into
// meta (bit-pattern maxima of non-negative floats: a NaN or inf anywhere wins, which invalidates the
// image -- see tc_meta_kernel).
__global__ void row_norms_kernel(const float* __restrict__ src0, const float* __restrict__ src1,
                                 long long row_stride, long long plane1_offset, long long n_rows,
                                 int dim, int k_total, int extra_steps, int sub_mode, float* __restrict__ bound,
                                 float* __restrict__ norm2, float* __restrict__ prefix, TcMeta* __restrict__ meta,
                                 const unsigned long long* __restrict__ guard) {
  // extra_steps: MMA k-steps beyond ceil(k_total / 16) (the L2 fold slots spilling into a k-step of
  // their own): their incoming accumulator is bounded by the full |x|^2
  if (guard_unchanged(guard)) return;
  const long long w = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= n_rows) return;
  const float* a = src0 + (size_t)w * row_stride;
  const float* b = src1 ? src1 + (size_t)w * row_stride : a + plane1_offset;
  double s = 0.0, sa = 0.0, sb = 0.0;   // s: running |x_{<= ...}|^2 (all lanes hold the same value)
  double p2 = 0.0;                      // sum of the squared prefix norms at the 16-element boundaries
  unsigned mx = 0u;
  for (int k0 = 0; k0 < k_total; k0 += 32) {
    const int k = k0 + lane;
    float x = 0.f;
    double xa = 0.0, xb = 0.0;
    if (k < k_total) {
      if (sub_mode) {
        x = k < dim ? __fsub_rn(b[k], a[k]) : 0.f;
        if (k < dim) { xa = (double)a[k] * (double)a[k]; xb = (double)b[k] * (double)b[k]; }
      } else {
        x = operand_value(a, b, dim, k, k_total);
      }
    }
    mx = max(mx, __float_as_uint(fabsf(x)));
    double h = (double)x * (double)x;   // -> sum over this lane's half-warp (one k-step)
#pragma unroll
    for (int o = 8; o > 0; o >>= 1) {
      h += __shfl_xor_sync(0xffffffffu, h, o);
      xa += __shfl_xor_sync(0xffffffffu, xa, o);
      xb += __shfl_xor_sync(0xffffffffu, xb, o);
    }
    const double h_lo = __shfl_sync(0xffffffffu, h, 0), h_hi = __shfl_sync(0xffffffffu, h, 16);
    sa += xa + __shfl_xor_sync(0xffffffffu, xa, 16);
    sb += xb + __shfl_xor_sync(0xffffffffu, xb, 16);
    s += h_lo;
    p2 += s;                                           // |x_{<= 16 i}|^2 after k-step i = 2 g + 1
    if (k0 + 16 < k_total) { s += h_hi; p2 += s; }     // ... and after k-step 2 g + 2
  }
  p2 += (double)extra_steps * s;
  mx = __reduce_max_sync(0xffffffffu, mx);
  if (lane == 0) {
    const float n2 = (float)s;
    norm2[w] = n2;
    // L2 head side: the reference rounds c + r before subtracting t, an error that scales with
    // |r| and |t| separately, so the bound uses |t| + |r| (>= |t - r|) for this operand
    const double nb = sub_mode ? sqrt(sa) + sqrt(sb) : sqrt(s);
    bound[w] = (float)(nb * (1.0 + 1e-6)) + 1e-30f;
    // the head-side operand t - r is bounded by |t| + |r| the same way: scale P by that ratio
    const double pr = sqrt(p2) * (s > 0.0 ? nb / sqrt(s) : 1.0);
    prefix[w] = (float)(pr * (1.0 + 1e-6)) + 1e-30f;
    atomicMax(reinterpret_cast<unsigned*>(&meta->max_abs), mx);
    atomicMax(reinterpret_cast<unsigned*>(&meta->max_norm2), __float_as_uint(fabsf(n2)));
  }
}

// Scales of one operand image, decided on the device from the maxima row_norms_kernel gathered.
//   bf16: scale = 1, phi = alpha = 1, S = 1, nothing else.
//   fp16: scale = 2^e with max|x| * scale in [2^8, 2^9): hi never overflows (65504), the lo part of
//         every element >= 2^-12 max|x| is a normal fp16 number (residual 2^-22 |x|); smaller elements
//         are off by <= 2^-25 in scaled units = 2^-33 max|x|, which sum_k |y_k| <= sqrt(K) |y| turns into
//         <= 2^-33 sqrt(K) max|x| |y| per pair: covered by adding kappa = 2^-11 sqrt(K) max|x| / 3 (+1 %)
//         to the row bounds (gamma >= 3 2^-22 multiplies them).
//         phi (candidate side, L2 fold): max_rows(|b|^2/2) * phi in [2^13, 2^14): the three pieces of
//         -|b|^2/2 * phi fit fp16 and are exact to 33 bits for every row within 2^-13 of the largest;
//         beyond, the absolute error 3 * 2^-25 / phi (|b|^2/2 units) goes into e_abs.
//         alpha (query side) = scale_a * scale_b / phi must itself be an fp16 normal power of two.
//   An operand with a NaN / inf entry, or whose alpha falls outside fp16, gets scale = NaN: its image,
//   S and hence both thresholds are NaN, every pair fails both tests and is rechecked exactly.
// maxima of the row bounds / running-magnitude factors over aligned blocks of 32 rows (rows past the
// table count as 0): one warp per block
__global__ void block_max_kernel(const float* __restrict__ bound, const float* __restrict__ prefix, long long n_rows,
                                 long long n_blocks, float* __restrict__ bmax, float* __restrict__ pmax,
                                 const unsigned long long* __restrict__ guard) {
  if (guard_unchanged(guard)) return;
  const long long w = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= n_blocks) return;
  const long long r = w * 32 + lane;
  const float x = r < n_rows ? bound[r] : 0.f, y = r < n_rows ? prefix[r] : 0.f;
  const unsigned mx = __reduce_max_sync(0xffffffffu, __float_as_uint(x));   // x, y >= 0 (NaN sorts on top)
  const unsigned my = __reduce_max_sync(0xffffffffu, __float_as_uint(y));
  if (lane == 0) { bmax[w] = __uint_as_float(mx); pmax[w] = __uint_as_float(my); }
}

__global__ void tc_meta_reset_kernel(TcMeta* __restrict__ m, const unsigned long long* __restrict__ guard) {
  if (guard_unchanged(guard)) return;
  if (threadIdx.x == 0) { m->max_abs = 0.f; m->max_norm2 = 0.f; }
}

// after a (re)build: remember which table content the image now holds
__global__ void tc_guard_commit_kernel(unsigned long long* __restrict__ guard) {
  if (threadIdx.x == 0) { guard[2] = guard[0]; guard[3] = guard[1]; }
}

// 128-bit content checksum of a table: two order-independent sums over its 64-bit words w_i,
//   h0 = sum w_i (2 i + 1),   h1 = sum (w_i ^ (w_i >> 31) ^ salt) (2 i + 1)        (mod 2^64)
// The odd, position-dependent multipliers make any single changed word change both sums, and several
// changed words cancel only by a 2^-64 coincidence per sum.  One pass at HBM speed: 16-byte loads,
// four in flight per thread.
__global__ void __launch_bounds__(256) table_checksum_kernel(const uint4* __restrict__ data, long long n_vec,
                                                             const uint32_t* __restrict__ tail_words,
                                                             int n_tail, unsigned long long salt,
                                                             unsigned long long* __restrict__ out) {
  unsigned long long h0 = 0ull, h1 = 0ull;
  auto add = [&](unsigned long long w, unsigned long long i) {
    const unsigned long long m = 2ull * i + 1ull;
    h0 += w * m;
    h1 += (w ^ (w >> 31) ^ salt) * m;
  };
  const long long stride = (long long)gridDim.x * blockDim.x;
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  for (; i + 3 * stride < n_vec; i += 4 * stride) {
    uint4 v[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) v[u] = __ldg(data + i + u * stride);
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const unsigned long long j = 2ull * (unsigned long long)(i + u * stride);
      add(((unsigned long long)v[u].y << 32) | v[u].x, j);
      add(((unsigned long long)v[u].w << 32) | v[u].z, j + 1ull);
    }
  }
  for (; i < n_vec; i += stride) {
    const uint4 v = __ldg(data + i);
    add(((unsigned long long)v.y << 32) | v.x, 2ull * (unsigned long long)i);
    add(((unsigned long long)v.w << 32) | v.z, 2ull * (unsigned long long)i + 1ull);
  }
  if (blockIdx.x == 0 && (int)threadIdx.x < n_tail)   // words past the last full 16-byte vector
    add(tail_words[threadIdx.x], 2ull * (unsigned long long)n_vec + threadIdx.x);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    h0 += __shfl_xor_sync(0xffffffffu, h0, o);
    h1 += __shfl_xor_sync(0xffffffffu, h1, o);
  }
  if ((threadIdx.x & 31) == 0) { atomicAdd(&out[0], h0); atomicAdd(&out[1], h1); }
}
__global__ void table_checksum_finish_kernel(unsigned long long* __restrict__ out) {
  if (threadIdx.x == 0) out[1] |= 1ull;   // never (0, 0): distinguishes "no image yet"
}

__global__ void tc_meta_kernel(TcMeta* __restrict__ m, const TcMeta* __restrict__ other, int k_total,
                               int is_query, int l2, int fp16, const unsigned long long* __restrict__ guard) {
  if (guard_unchanged(guard)) return;
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  const float mx = m->max_abs, n2 = m->max_norm2;
  const bool finite = mx <= 3.0e38f && n2 <= 3.0e38f;   // false for NaN and inf
  float scale = 1.f, fold = 1.f, kappa = 0.f, acc = 1.f, e_abs = 0.f;
  bool ok = finite;
  if (fp16 && finite) {
    if (mx > 0.f) {
      int ex; frexpf(mx, &ex);                 // mx = f * 2^ex, f in [0.5, 1)
      int e = 9 - ex;
      e = max(-120, min(120, e));
      scale = ldexpf(1.f, e);
      kappa = mx * 0x1p-11f * sqrtf((float)k_total) * (1.01f / 3.f);
    }
    if (!is_query && l2 && n2 > 0.f) {
      int ex; frexpf(0.5f * n2, &ex);
      fold = ldexpf(1.f, max(-120, min(120, 14 - ex)));   // phi
    }
  }
  if (is_query) {
    const float sb = other->scale, phi = other->fold;
    acc = scale * sb;                                      // NaN if the table image is invalid
    if (l2) {
      fold = acc / phi;                                    // alpha
      if (fp16) {
        if (!(fold >= 0x1p-14f && fold <= 0x1p15f)) ok = false;
        e_abs = 0x1p-22f / phi;                            // 8 * 2^-25 / phi: fold pieces, score = 2 f - |a|^2
      }
    }
    if (!(acc >= 0x1p-60f && acc <= 0x1p60f)) ok = false;
  }
  const float nanv = __uint_as_float(0x7fc00000u);
  m->scale = ok ? scale : nanv;
  m->fold = ok ? fold : nanv;
  m->acc_scale = ok ? acc : nanv;
  m->e_abs = e_abs;
  m->kappa = kappa;
}

template <int EL>
__global__ void recheck_kernel(int dim, const unsigned long long* __restrict__ region_counts,
                               unsigned long long region_cap, const int2* __restrict__ pairs,
                               const float* __restrict__ qplain, const float* __restrict__ ent0,
                               const float* __restrict__ ent1, const float* __restrict__ s_true,
                               int32_t* __restrict__ counts) {
  constexpr int QW = ElemTraits<EL>::QW, CW = ElemTraits<EL>::CW;
  constexpr bool NORM = ElemTraits<EL>::RED == RED_NORM2;
  constexpr int PAIRS_PER_WARP = NORM ? 4 : 1;
  const unsigned long long region = blockIdx.y;
  const unsigned long long n_pairs = min(region_counts[region], region_cap);
  const int lane = threadIdx.x & 31;
  const unsigned long long warp_global = ((unsigned long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const unsigned long long n_warps = ((unsigned long long)gridDim.x * blockDim.x) >> 5;
  const int2* list = pairs + region * region_cap;
  if (!NORM && dim < 8) {  // one-lane schedule: plain per-thread scorer
    for (unsigned long long i = warp_global * 32 + lane; i < n_pairs; i += n_warps * 32) {
      const int2 pr = list[i];
      const float* q0 = qplain + (size_t)pr.x * QW * dim;
      const float* c0 = ent0 + (size_t)pr.y * dim;
      const float* c1 = (CW == 3 ? ent1 + (ent1 - ent0) : (CW == 2 ? ent1 : ent0)) + (size_t)pr.y * dim;
      const float* cm = (CW == 3 ? ent1 : ent0) + (size_t)pr.y * dim;   // middle plane (three-plane kinds)
      if (pair_score_natural<EL>(dim, q0, q0 + (size_t)(QW - 1) * dim, c0, c1, q0 + (size_t)(QW / 2) * dim, cm) >=
          s_true[pr.x])
        atomicAdd(&counts[pr.x], 1);
    }
    return;
  }
  for (unsigned long long base = warp_global * PAIRS_PER_WARP; base < n_pairs; base += n_warps * PAIRS_PER_WARP) {
    const unsigned long long i = base + (NORM ? (lane >> 3) : 0);
    const bool valid = i < n_pairs;
    const int2 pr = list[valid ? i : base];  // idle groups redo the first pair (shuffles stay uniform)
    const float* q0 = qplain + (size_t)pr.x * QW * dim;
    const float* q1 = q0 + (size_t)(QW - 1) * dim;
    const float* c0 = ent0 + (size_t)pr.y * dim;
    const float* c1 = (CW == 3 ? ent1 + (ent1 - ent0) : (CW == 2 ? ent1 : ent0)) + (size_t)pr.y * dim;
    const float* qm = q0 + (size_t)(QW / 2) * dim;                      // middle plane (three-plane kinds)
    const float* cm = (CW == 3 ? ent1 : ent0) + (size_t)pr.y * dim;
    const float sc = pair_score_chains<EL>(dim, q0, q1, c0, c1, lane, qm, cm);
    const bool leader = NORM ? ((lane & 7) == 0) : (lane == 0);
    if (valid && leader && sc >= s_true[pr.x]) atomicAdd(&counts[pr.x], 1);
  }
}

// stats[0] = near-tie pairs found (or capacity + 1 if any region overflowed), stats[1] = capacity
__global__ void tc_stats_kernel(const unsigned long long* __restrict__ region_counts, int regions,
                                unsigned long long region_cap, unsigned long long* __restrict__ stats) {
  unsigned long long total = 0;
  bool over = false;
  for (int r = 0; r < regions; ++r) {
    total += region_counts[r];
    over |= region_counts[r] > region_cap;
  }
  const unsigned long long cap = region_cap * (unsigned long long)regions;
  stats[0] = over ? cap + 1 : total;
  stats[1] = cap;
}

}  // namespace

// ------------------------------------------------------------------------------------------
// Geometry choice.  k-block = 32 bf16 (64-byte swizzle) by default: finer stages, 7 % instead of
// 23 % padding at k = 200, and the query tile's A image (<= 7 blocks, k_total <= 224) can stay
// resident in shared memory so that only B streams (1/3 less L2 -> SM traffic, the limiter of
// the streamed form).  KGE_TC_BK=64 selects the 128-byte-swizzle layout (2 stages of 96 KB),
// KGE_TC_RESIDENT=0 disables residency, KGE_TC_GROUP sets candidate tiles per unit.
// ------------------------------------------------------------------------------------------
namespace {
int env_int(const char* name, int dflt) {
  const char* v = getenv(name);
  return (v && *v) ? atoi(v) : dflt;
}
struct Config {
  int bk, resident, group, max_ctas, fp16;
  Config()
      : bk(env_int("KGE_TC_BK", 32) == 64 ? 64 : 32), resident(env_int("KGE_TC_RESIDENT", 1) != 0),
        group(env_int("KGE_TC_GROUP", 0)), max_ctas(env_int("KGE_TC_MAX_CTAS", 0)),
        fp16(env_int("KGE_TC_FP16", 1) != 0) {}
};
Config& config() {
  static Config c;
  return c;
}
}  // namespace

void configure(int bk_, int resident_, int group_, int max_ctas_, int fp16_) {
  Config& c = config();
  if (bk_ == 32 || bk_ == 64) c.bk = bk_;
  if (resident_ >= 0) c.resident = resident_ != 0;
  if (group_ >= 0) c.group = group_;
  if (max_ctas_ >= 0) c.max_ctas = max_ctas_;
  if (fp16_ >= 0) c.fp16 = fp16_ != 0;
}
bool fp16() { return config().fp16 != 0; }
int bk() { return config().bk; }
int n_kblocks(int k_total) { return (k_total + bk() - 1) / bk(); }
bool resident(int n_kb) {
  return config().resident && bk() == 32 && n_kb <= 7 && smem_bytes<32, true>(n_kb) <= SMEM_LIMIT;
}
int ct_group(int n_kb) {
  if (config().group > 0) return config().group;
  return resident(n_kb) ? 32 : 16;
}
// With few query tiles (a rank's slice of a query-sharded run) whole groups of 32 candidate tiles
// are too coarse a unit for one CTA per SM: shrink the group until there are >= 32 units per CTA.
int ct_group_for(int n_kb, long long n_qt, long long n_ct, int sms) {
  int g = ct_group(n_kb);
  if (config().group > 0) return g;
  while (g > 4 && n_qt * ((n_ct + g - 1) / g) < 32ll * sms) g >>= 1;
  return g;
}

size_t a_image_bytes(long long n_q, int n_kb) {
  const long long n_qt = (n_q + BM - 1) / BM;
  return (size_t)n_qt * n_kb * 2 * BM * 2 * bk();
}
size_t b_image_bytes(long long n_rows, int n_kb) {
  const long long n_ct = (n_rows + BN - 1) / BN;
  return (size_t)n_ct * n_kb * 2 * BN * 2 * bk();
}

namespace {
template <int ROWS>
void launch_pack_operand(const float* src0, const float* src1, long long row_stride, long long plane1_offset,
                         long long n_rows, int dim, int k_total, int n_kb, int sub_mode, int fold,
                         const float* norm2, const TcMeta* meta, const unsigned long long* guard,
                         unsigned char* out, cudaStream_t st) {
  const long long n_tiles = (n_rows + ROWS - 1) / ROWS;
  const long long total = n_tiles * n_kb * ROWS * (bk() / 8);
  const unsigned blocks = (unsigned)((total + 255) / 256);
#define KGE_PACK(BKT, F16)                                                                              \
  pack_operand_kernel<ROWS, BKT, F16><<<blocks, 256, 0, st>>>(src0, src1, row_stride, plane1_offset, n_rows, dim, \
                                                              k_total, n_kb, sub_mode, fold, norm2, meta, guard, out)
  if (bk() == 64) { if (fp16()) KGE_PACK(64, true); else KGE_PACK(64, false); }
  else { if (fp16()) KGE_PACK(32, true); else KGE_PACK(32, false); }
#undef KGE_PACK
}
}  // namespace


cudaError_t launch_pack_b(const float* ent0, const float* ent1, long long n_rows, int dim, int k_total,
                          int n_kb, bool fold, unsigned char* bpack, float* cbound, float* cnorm2, float* cprefix,
                          float* cbmax32, float* cpmax32, TcMeta* meta_b, unsigned long long* guard, cudaStream_t st) {
  if (n_rows <= 0) return cudaSuccess;
  if (guard) {
    // checksum of the table as it is now (one pass over it at HBM speed); if it equals the one the
    // image was built from, every kernel below returns immediately
    cudaError_t e = cudaMemsetAsync(guard, 0, 2 * sizeof(unsigned long long), st);
    if (e != cudaSuccess) return e;
    const long long n_words = n_rows * dim;
    auto checksum = [&](const float* tab, unsigned long long salt) {
      // 16-byte vector loads over the aligned middle of the table; the <= 3 words before it and the
      // <= 3 words after it go through the kernel's tail path (positions past the vector part)
      const uint32_t* words = reinterpret_cast<const uint32_t*>(tab);
      const long long head = min(n_words, (long long)(((16u - (reinterpret_cast<uintptr_t>(tab) & 15u)) & 15u) / 4u));
      const long long n_vec = (n_words - head) / 4;
      const int n_tail = (int)(n_words - head - 4 * n_vec);
      const unsigned blocks = (unsigned)max(1ll, min((n_vec + 1023) / 1024, (long long)132 * 8));   // 8 per H100 SM
      table_checksum_kernel<<<blocks, 256, 0, st>>>(reinterpret_cast<const uint4*>(words + head), n_vec,
                                                    words + head + 4 * n_vec, n_tail, salt, guard);
      if (head > 0)
        table_checksum_kernel<<<1, 32, 0, st>>>(nullptr, 0, words, (int)head, salt ^ 0xA5A5A5A5A5A5A5A5ull, guard);
    };
    checksum(ent0, 0ull);
    if (ent1) checksum(ent1, 0x5851F42D4C957F2Dull);
    if (ent1 && !fold && k_total == 3 * dim) checksum(ent1 + (ent1 - ent0), 0x2545F4914F6CDD1Dull);   // third plane
    table_checksum_finish_kernel<<<1, 32, 0, st>>>(guard);
  }
  tc_meta_reset_kernel<<<1, 32, 0, st>>>(meta_b, guard);
  // norms first: with fold the image carries -|b|^2/2 (the SAME fp32 value the bound uses)
  row_norms_kernel<<<(unsigned)((n_rows * 32 + 255) / 256), 256, 0, st>>>(
      ent0, ent1, dim, 0, n_rows, dim, fold ? dim : k_total, fold ? (k_total + 15) / 16 - (dim + 15) / 16 : 0, 0,
      cbound, cnorm2, cprefix, meta_b, guard);
  {
    const long long n_blocks = ((n_rows + BN - 1) / BN) * (BN / 32);
    block_max_kernel<<<(unsigned)((n_blocks * 32 + 255) / 256), 256, 0, st>>>(cbound, cprefix, n_rows, n_blocks, cbmax32,
                                                                              cpmax32, guard);
  }
  tc_meta_kernel<<<1, 32, 0, st>>>(meta_b, nullptr, k_total, 0, fold ? 1 : 0, fp16() ? 1 : 0, guard);
  launch_pack_operand<BN>(ent0, ent1, dim, 0, n_rows, dim, k_total, n_kb, 0, fold ? 2 : 0, cnorm2, meta_b, guard,
                          bpack, st);
  if (guard) tc_guard_commit_kernel<<<1, 32, 0, st>>>(guard);
  return cudaGetLastError();
}

cudaError_t launch_pack_a(const float* qplain, int qw, long long n_q, int dim, int k_total, int n_kb,
                          int sub_mode, bool fold, unsigned char* apack, float* qbound, float* qnorm2, float* qprefix,
                          TcMeta* meta_a, const TcMeta* meta_b, cudaStream_t st) {
  if (n_q <= 0) return cudaSuccess;
  tc_meta_reset_kernel<<<1, 32, 0, st>>>(meta_a, nullptr);
  // qplain rows are [qw][dim]: plane 1 (if any) follows plane 0 inside the row
  row_norms_kernel<<<(unsigned)((n_q * 32 + 255) / 256), 256, 0, st>>>(
      qplain, nullptr, (long long)qw * dim, dim, n_q, dim, fold ? dim : k_total,
      fold ? (k_total + 15) / 16 - (dim + 15) / 16 : 0, sub_mode, qbound, qnorm2, qprefix, meta_a, nullptr);
  tc_meta_kernel<<<1, 32, 0, st>>>(meta_a, meta_b, k_total, 1, fold ? 1 : 0, fp16() ? 1 : 0, nullptr);
  launch_pack_operand<BM>(qplain, nullptr, (long long)qw * dim, dim, n_q, dim, k_total, n_kb, sub_mode,
                          fold ? 1 : 0, nullptr, meta_a, nullptr, apack, st);
  return cudaGetLastError();
}

namespace {
template <bool L2, bool DUMP, bool F16, int BKT, bool RES>
cudaError_t launch_kernel(const TcScanParams& p, int grid, size_t smem, cudaStream_t st) {
  constexpr auto kernel = tc_scan_kernel<L2, DUMP, F16, BKT, RES>;
  const cudaError_t e = set_attribute_once<kernel>(cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_LIMIT);
  if (e != cudaSuccess) return e;
  kernel<<<grid, THREADS, smem, st>>>(p);
  return cudaGetLastError();
}

template <int BKT, bool RES, bool F16>
cudaError_t launch_variant(const TcScanParams& p, int grid, cudaStream_t st) {
  const size_t smem = smem_bytes<BKT, RES>(p.n_kb);
  if (smem > SMEM_LIMIT) return cudaErrorInvalidValue;
  if (p.dump)
    return p.l2 ? launch_kernel<true, true, F16, BKT, RES>(p, grid, smem, st)
                : launch_kernel<false, true, F16, BKT, RES>(p, grid, smem, st);
  return p.l2 ? launch_kernel<true, false, F16, BKT, RES>(p, grid, smem, st)
              : launch_kernel<false, false, F16, BKT, RES>(p, grid, smem, st);
}

template <bool F16>
cudaError_t launch_format(const TcScanParams& p, int grid, cudaStream_t st) {
  if (bk() == 64) return launch_variant<64, false, F16>(p, grid, st);
  if (resident(p.n_kb)) return launch_variant<32, true, F16>(p, grid, st);
  return launch_variant<32, false, F16>(p, grid, st);
}
}  // namespace

cudaError_t launch_tc_scan(const TcScanParams& p_in, cudaStream_t st) {
  TcScanParams p = p_in;
  p.fp16 = fp16() ? 1 : 0;
  const int grid = scan_grid_size(p.n_q, p.n_rows, p.n_kb, &p.ct_group);
  if (grid <= 0) return cudaSuccess;
  return p.fp16 ? launch_format<true>(p, grid, st) : launch_format<false>(p, grid, st);
}

cudaError_t launch_recheck(int el, int dim, const unsigned long long* region_counts, int regions,
                           unsigned long long region_cap, const int2* pairs, const float* qplain,
                           const float* ent0, const float* ent1, const float* s_true, int32_t* counts,
                           unsigned long long* stats, cudaStream_t st) {
  if (regions <= 0 || region_cap == 0) return cudaSuccess;
  dim3 grid(96, (unsigned)regions);
#define CALL_RC(EL) \
  recheck_kernel<EL><<<grid, 128, 0, st>>>(dim, region_counts, region_cap, pairs, qplain, ent0, ent1, s_true, counts)
  switch (el) {
    case EL_DOT1: CALL_RC(EL_DOT1); break;
    case EL_DOT2: CALL_RC(EL_DOT2); break;
    case EL_DOT3: CALL_RC(EL_DOT3); break;
    case EL_L2_TAIL: CALL_RC(EL_L2_TAIL); break;
    case EL_L2_HEAD: CALL_RC(EL_L2_HEAD); break;
    case EL_ROT: CALL_RC(EL_ROT); break;
    default: return cudaErrorInvalidValue;
  }
#undef CALL_RC
  if (stats) tc_stats_kernel<<<1, 1, 0, st>>>(region_counts, regions, region_cap, stats);
  return cudaGetLastError();
}

int scan_grid_size(long long n_q, long long n_rows, int n_kb, int* group_out) {
  int dev = 0, sms = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 0;
  if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) return 0;
  const long long n_qt = (n_q + BM - 1) / BM, n_ct = (n_rows + BN - 1) / BN;
  if (config().max_ctas > 0 && config().max_ctas < sms) sms = config().max_ctas;
  const long long g = ct_group_for(n_kb, n_qt, n_ct, sms);
  if (group_out) *group_out = (int)g;
  const long long units = n_qt * ((n_ct + g - 1) / g);
  return (int)(units < sms ? units : sms);
}

}  // namespace tc
}  // namespace kge
