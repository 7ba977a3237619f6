// extern "C" entry points of libkge_b200.so (declared in include/kge_b200.h).
#include <mutex>
#include <map>
#include <memory>
#include <optional>
#include <stdio.h>
#include <string.h>
#include <vector>

#include "../../include/kge_b200.h"
#include "kernels.h"
#include "schedule.h"
#include "tc.h"
#include "train.h"

namespace {

thread_local char g_err[512] = "";

int fail(int code, const char* msg) {
  snprintf(g_err, sizeof(g_err), "%s", msg);
  return code;
}

// "fn: what", the form of every argument error of the entry points
int fail(int code, const char* fn, const char* what) {
  snprintf(g_err, sizeof(g_err), "%s: %s", fn, what);
  return code;
}

int fail_cuda(cudaError_t e, const char* where) {
  snprintf(g_err, sizeof(g_err), "%s: %s", where, cudaGetErrorString(e));
  return KGE_ERR_CUDA;
}

#define KGE_CUDA_TRY(expr, where)                      \
  do {                                                 \
    cudaError_t _e = (expr);                           \
    if (_e != cudaSuccess) return fail_cuda(_e, where); \
  } while (0)

// The kernels are launched on the CURRENT device with the stream the caller hands in; a caller whose
// current device is not the one its buffers live on (a model on cuda:1 while cuda:0 is current)
// would otherwise launch on the wrong device.  Every launching entry point therefore switches to
// the device that owns its first device pointer for the duration of the call.
struct DeviceScope {
  int prev = -1;
  bool switched = false;
  explicit DeviceScope(const void* device_ptr) {
    if (!device_ptr) return;
    cudaPointerAttributes at;
    if (cudaPointerGetAttributes(&at, device_ptr) != cudaSuccess) { cudaGetLastError(); return; }
    if (at.type != cudaMemoryTypeDevice && at.type != cudaMemoryTypeManaged) return;
    if (cudaGetDevice(&prev) != cudaSuccess) return;
    if (prev != at.device && cudaSetDevice(at.device) == cudaSuccess) switched = true;
  }
  ~DeviceScope() {
    if (switched) cudaSetDevice(prev);
  }
};

struct HostSchedule {
  kge::Schedule s;
  std::vector<int32_t> inv_perm;
};

// Schedules depend on (reduce kind, dim) only; building one is O(dim).  Cached per process.
const HostSchedule* get_schedule(int model, int dim) {
  static std::mutex mu;
  static std::map<std::pair<int, int>, std::unique_ptr<HostSchedule>> cache;
  const int kind = kge::reduce_kind_for_model(model);
  if (kind < 0) return nullptr;
  std::lock_guard<std::mutex> lock(mu);
  auto key = std::make_pair(kind, dim);
  auto it = cache.find(key);
  if (it != cache.end()) return it->second.get();
  auto hs = std::make_unique<HostSchedule>();
  if (!kge::build_schedule(kind, dim, &hs->s)) return nullptr;
  hs->inv_perm.assign(dim, 0);
  for (int pos = 0; pos < dim; ++pos) hs->inv_perm[hs->s.perm[pos]] = pos;
  const HostSchedule* out = hs.get();
  cache[key] = std::move(hs);
  return out;
}

size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// Bump allocator over a caller's workspace: 256-byte aligned pieces from `off` on; base = nullptr
// only sizes them.
struct Carver {
  void* base;
  size_t off = 0;
  template <class T>
  T* take(size_t bytes) {
    void* p = base ? static_cast<char*>(base) + off : nullptr;
    off += align_up(bytes, 256);
    return static_cast<T*>(p);
  }
};

// Workspace carve-up shared by kge_rank_side, kge_filter_side, kge_score_all and kge_topk_side.
struct Workspace {
  float* qplain;
  float* qpacked;
  float* s_true;
  int32_t* perm;
  uint8_t* code;
  // tensor-core path
  unsigned char* apack = nullptr;
  float* qbound = nullptr;
  float* qnorm2 = nullptr;
  float* qprefix = nullptr;
  kge::tc::TcMeta* meta_a = nullptr;
  // near-tie list (tensor-core and approximate scans)
  unsigned long long* amb_count = nullptr;
  int2* amb_pairs = nullptr;
  unsigned long long amb_cap = 0;
  size_t bytes;
};

bool tc_supported(int el) {
  return el == kge::EL_DOT1 || el == kge::EL_DOT2 || el == kge::EL_DOT3 || el == kge::EL_L2_TAIL ||
         el == kge::EL_L2_HEAD;
}
bool tc_is_l2(int el) { return el == kge::EL_L2_TAIL || el == kge::EL_L2_HEAD; }
// bound-and-refine on the fp32 pipes (approximate element arithmetic + exact recheck): RotatE
bool approx_supported(int el) { return el == kge::EL_ROT; }
// Byte offsets inside a tensor-core candidate image (kge_tc_pack_table): operand planes, then per-row
// norm bounds / squared norms / running-magnitude factors (padded to whole 256-row tiles), then the
// maxima of the bounds and of the factors over aligned blocks of 32 rows (what one epilogue warp
// needs per 32-column block), then the TcMeta record.
struct TcImageLayout {
  size_t cbound, cnorm2, cprefix, cbmax32, cpmax32, meta, total;
  TcImageLayout(int64_t n_rows, int n_kb) {
    const size_t n_ct = (size_t)((n_rows + kge::tc::TC_BN - 1) / kge::tc::TC_BN);
    const size_t rows = n_ct * kge::tc::TC_BN * sizeof(float);
    cbound = kge::tc::b_image_bytes(n_rows, n_kb);
    cnorm2 = cbound + rows;
    cprefix = cnorm2 + rows;
    cbmax32 = cprefix + rows;
    cpmax32 = cbmax32 + rows / 32;
    meta = align_up(cpmax32 + rows / 32, 256);
    total = meta + kge::tc::TC_META_BYTES;
  }
};
// The pieces of a candidate image at `bpack`, typed: writable for the pack (Byte = unsigned char),
// read-only for the scan (Byte = const unsigned char).
template <class Byte>
struct TcImage {
  template <class T>
  using Ptr = std::conditional_t<std::is_const<Byte>::value, const T*, T*>;
  Byte* bpack;
  Ptr<float> cbound, cnorm2, cprefix, cbmax32, cpmax32;
  Ptr<kge::tc::TcMeta> meta;
  TcImage(Byte* base, int64_t n_rows, int n_kb) : bpack(base) {
    const TcImageLayout L(n_rows, n_kb);
    auto at = [&](size_t off) { return reinterpret_cast<Ptr<float>>(base + off); };
    cbound = at(L.cbound); cnorm2 = at(L.cnorm2); cprefix = at(L.cprefix);
    cbmax32 = at(L.cbmax32); cpmax32 = at(L.cpmax32);
    meta = reinterpret_cast<Ptr<kge::tc::TcMeta>>(base + L.meta);
  }
};
// contraction length of the operand images: all planes for ComplEx / Analogy; L2 carries the candidate's
// squared norm in three extra k slots (tc.h: launch_pack_b)
int tc_k_total(int el, int dim) {
  if (el == kge::EL_DOT3) return 3 * dim;   // all three planes of Analogy
  return el == kge::EL_DOT2 ? 2 * dim : (tc_is_l2(el) ? dim + 3 : dim);
}

Workspace carve(void* base, int qw, int dim, int64_t n, int el = -1, int64_t n_rows = 0, int flags = 0) {
  const int64_t n_qt = (n + kge::TILE_Q - 1) / kge::TILE_Q;
  Carver c{base};
  Workspace w;
  w.qplain = c.take<float>((size_t)n * qw * dim * sizeof(float));
  w.qpacked = c.take<float>((size_t)n_qt * dim * qw * kge::TILE_Q * sizeof(float));
  w.s_true = c.take<float>((size_t)n_qt * kge::TILE_Q * sizeof(float));
  w.perm = c.take<int32_t>((size_t)dim * sizeof(int32_t));
  w.code = c.take<uint8_t>((size_t)dim);
  const bool want_tc = (flags & KGE_FLAG_TENSOR_CORE) && el >= 0 && tc_supported(el) && n_rows > 0;
  const bool want_approx = (flags & KGE_FLAG_APPROX_SCAN) && approx_supported(el) && n_rows > 0;
  if (want_tc) {
    const int n_kb = kge::tc::n_kblocks(tc_k_total(el, dim));
    w.apack = c.take<unsigned char>(kge::tc::a_image_bytes(n, n_kb));
    w.qbound = c.take<float>((size_t)n * sizeof(float));
    w.qnorm2 = c.take<float>((size_t)n * sizeof(float));
    w.qprefix = c.take<float>((size_t)n * sizeof(float));
    w.meta_a = c.take<kge::tc::TcMeta>(kge::tc::TC_META_BYTES);
  }
  if (want_tc || want_approx) {
    const int64_t n_tc_qt = (n + kge::tc::TC_BM - 1) / kge::tc::TC_BM;
    w.amb_count = c.take<unsigned long long>((size_t)n_tc_qt * sizeof(unsigned long long));
    // near-tie list, one region per query tile: room for 1/128 of all pairs (the band is
    // 0.1-0.3 % on average), at least 8 Ki entries per tile, at most 256 Mi in total
    unsigned long long cap = (unsigned long long)n * (unsigned long long)n_rows / 128ull;
    if (cap < (unsigned long long)n_tc_qt * 8192ull) cap = (unsigned long long)n_tc_qt * 8192ull;
    if (cap > (1ull << 28)) cap = 1ull << 28;
    w.amb_cap = cap;
    w.amb_pairs = c.take<int2>((size_t)cap * sizeof(int2));
  }
  w.bytes = c.off;
  return w;
}

// Steps shared by ranking and dense scoring: upload the schedule, build the query vectors.
int prepare_queries(int model, int side, int dim, int64_t n, const float* hrows,
                    const float* trows, const float* rel0, const float* rel1,
                    const int64_t* r_idx, const HostSchedule* hs, const Workspace& w, int el,
                    cudaStream_t stream, bool scalar_layout = true) {
  KGE_CUDA_TRY(cudaMemcpyAsync(w.perm, hs->s.perm.data(), (size_t)dim * sizeof(int32_t),
                               cudaMemcpyHostToDevice, stream),
               "upload schedule perm");
  KGE_CUDA_TRY(cudaMemcpyAsync(w.code, hs->s.code.data(), (size_t)dim, cudaMemcpyHostToDevice,
                               stream),
               "upload schedule code");
  KGE_CUDA_TRY(kge::launch_prep_queries(model, side, dim, n, hrows, trows, rel0, rel1, r_idx,
                                        w.qplain, stream),
               "prep_queries");
  if (scalar_layout)   // the k-major query image of the scalar scan (the tensor-core scan builds its own)
    KGE_CUDA_TRY(kge::launch_pack_queries(w.qplain, kge::elem_qw(el), dim, n, w.perm, w.qpacked,
                                          stream),
                 "pack_queries");
  return KGE_OK;
}

bool model_needs_rel1(int model) { return model == KGE_COMPLEX || model == KGE_ROTATE || model == KGE_ANALOGY; }

// Optional CUDA-event bracketing of the scan launches (kge_scan_timing_*).
std::mutex g_timing_mu;
bool g_timing_on = false;
constexpr int TIMING_KINDS = 3;  // 0 scalar scan, 1 tensor-core scan, 2 exact recheck of near-ties
std::vector<std::pair<cudaEvent_t, cudaEvent_t>> g_timing_events[TIMING_KINDS];

template <class Launch>
cudaError_t timed_launch(int kind, cudaStream_t st, Launch&& launch) {
  bool on;
  {
    std::lock_guard<std::mutex> lock(g_timing_mu);
    on = g_timing_on;
  }
  if (!on) return launch();
  cudaEvent_t a, b;
  cudaError_t e = cudaEventCreate(&a);
  if (e != cudaSuccess) return e;
  e = cudaEventCreate(&b);
  if (e != cudaSuccess) return e;
  cudaEventRecord(a, st);
  e = launch();
  cudaEventRecord(b, st);
  std::lock_guard<std::mutex> lock(g_timing_mu);
  g_timing_events[kind].emplace_back(a, b);
  return e;
}

cudaError_t timed_scan(int el, bool casc, const kge::ScanParams& p, cudaStream_t st) {
  return timed_launch(0, st, [&] { return kge::launch_scan(el, casc, p, st); });
}

// The setup kge_rank_side, kge_score_all and kge_topk_side share, over their argument structs (which
// name the shared fields alike).  Each entry point runs checks of its own between these steps; that
// order decides which error a call with several bad arguments gets.
template <class Args>
struct QueryCall {
  const char* fn;
  const Args* a;
  int el = -1;
  const HostSchedule* hs = nullptr;
  std::optional<DeviceScope> device;

  int error(int code, const char* what) const { return fail(code, fn, what); }
  int lookup_kind() {
    el = kge::elem_kind_for(a->model, a->side);
    return el < 0 ? error(KGE_ERR_ARG, "unknown model/side") : KGE_OK;
  }
  // the query tables and the workspace; own_ok: the pointers only this entry point requires
  int check_tables(bool own_ok, bool ent1_missing = false) const {
    const bool rel_side = a->side == KGE_SIDE_REL;  // candidates = relation rows; rel0 / rel1 unused
    if (!own_ok || (!a->rel0 && !rel_side) || !a->hrows || !a->trows || !a->workspace)
      return error(KGE_ERR_ARG, "null pointer");
    if (ent1_missing) return error(KGE_ERR_ARG, "ent1 required");
    if (!rel_side && model_needs_rel1(a->model) && !a->rel1) return error(KGE_ERR_ARG, "rel1 required");
    return KGE_OK;
  }
  int lookup_schedule() {
    hs = get_schedule(a->model, a->dim);
    return hs ? KGE_OK : error(KGE_ERR_UNSUPPORTED, "unsupported dim");
  }
  // On the device of `device_ptr` for the rest of the call: check the size of the carved workspace,
  // upload the schedule and build the queries.
  int prepare(const void* device_ptr, const Workspace& w, size_t bytes, bool scalar_layout = true) {
    device.emplace(device_ptr);
    if (bytes > a->workspace_bytes) return error(KGE_ERR_ARG, "workspace too small");
    return prepare_queries(a->model, a->side, a->dim, a->n, a->hrows, a->trows, a->rel0, a->rel1, a->r_idx, hs, w,
                           el, stream(), scalar_layout);
  }
  cudaStream_t stream() const { return static_cast<cudaStream_t>(a->stream); }
};

// The scalar scan of n_q queries (qpacked) against n_rows candidates (packed); the caller sets what
// it produces: counts, scores, the near-tie list or the collect lists.
kge::ScanParams scan_params(const float* packed, const float* qpacked, const float* s_true, const HostSchedule* hs,
                            int dim, int64_t n_q, int64_t n_rows) {
  kge::ScanParams p;
  p.packed = packed;
  p.qpacked = qpacked;
  p.s_true = s_true;
  p.code_host = hs->s.code.data();
  p.dim = dim;
  p.n_q = n_q;
  p.n_rows = n_rows;
  p.n_ct = (n_rows + kge::TILE_C - 1) / kge::TILE_C;
  p.n_qt = (n_q + kge::TILE_Q - 1) / kge::TILE_Q;
  return p;
}

// Bound-and-refine, the tensor-core scan (tc) or RotatE's approximate scan: scan(region_cap) decides
// every pair outside the near-tie band and lists the rest, one region per 128-query tile; the
// recheck re-scores those exactly.
template <class Scan>
int refine(bool tc, const kge_rank_args_t* a, int el, const Workspace& w, cudaStream_t st, Scan&& scan) {
  const int regions = (int)((a->n + kge::tc::TC_BM - 1) / kge::tc::TC_BM);
  const unsigned long long region_cap = w.amb_cap / (unsigned long long)regions;
  KGE_CUDA_TRY(cudaMemsetAsync(w.amb_count, 0, (size_t)regions * sizeof(unsigned long long), st),
               tc ? "tc reset list" : "approx reset list");
  KGE_CUDA_TRY(timed_launch(tc ? 1 : 0, st, [&] { return scan(region_cap); }), tc ? "tc scan" : "approx rank scan");
  KGE_CUDA_TRY(timed_launch(2, st, [&] {
                 return kge::tc::launch_recheck(el, a->dim, w.amb_count, regions, region_cap, w.amb_pairs, w.qplain,
                                                a->ent0, a->ent1, w.s_true, a->raw_count,
                                                reinterpret_cast<unsigned long long*>(a->tc_stats), st);
               }),
               tc ? "tc recheck" : "approx recheck");
  return KGE_OK;
}

// The sparse filter pass over the CSR of `a`, after either scan
cudaError_t launch_filter_pass(const kge_rank_args_t* a, int el, bool casc, const Workspace& w, cudaStream_t st) {
  return kge::launch_filter(el, casc, a->dim, a->n, a->n_filt, w.qplain, a->ent0, a->ent1, a->ent_lo, a->n_rows,
                            a->filt_offs, a->filt_ids, a->filt_qid, w.perm, w.code, w.s_true, a->filt_sub, st);
}

}  // namespace

extern "C" {

int kge_abi_version(void) { return KGE_ABI_VERSION; }

const char* kge_last_error(void) { return g_err; }

int kge_cand_planes(int model) {
  const int el = kge::elem_kind_for(model, KGE_SIDE_TAIL);
  return el < 0 ? 0 : kge::elem_cw(el);
}

int kge_query_planes(int model, int side) {
  const int el = kge::elem_kind_for(model, side);
  return el < 0 ? 0 : kge::elem_qw(el);
}

int kge_build_schedule(int model, int dim, int32_t* perm_host, uint8_t* code_host) {
  if (!perm_host || !code_host) return fail(KGE_ERR_ARG, "kge_build_schedule: null output");
  const HostSchedule* hs = get_schedule(model, dim);
  if (!hs) return fail(KGE_ERR_UNSUPPORTED, "kge_build_schedule: unsupported model or dim");
  memcpy(perm_host, hs->s.perm.data(), (size_t)dim * sizeof(int32_t));
  memcpy(code_host, hs->s.code.data(), (size_t)dim);
  return KGE_OK;
}

int kge_schedule_depth(int model, int dim) {
  const HostSchedule* hs = get_schedule(model, dim);
  return hs ? kge::schedule_depth(hs->s) : -1;
}

size_t kge_packed_table_floats(int model, int64_t n_rows, int dim) {
  const int planes = kge_cand_planes(model);
  if (planes == 0 || n_rows < 0 || dim < 1) return 0;
  const int64_t n_ct = (n_rows + kge::TILE_C - 1) / kge::TILE_C;
  return (size_t)n_ct * dim * planes * kge::TILE_C;
}

int kge_pack_table(int model, const float* ent0, const float* ent1, int64_t n_rows, int dim,
                   float* packed, void* stream) {
  const int planes = kge_cand_planes(model);
  if (planes == 0) return fail(KGE_ERR_ARG, "kge_pack_table: unknown model");
  if (!ent0 || !packed || (planes >= 2 && !ent1))
    return fail(KGE_ERR_ARG, "kge_pack_table: null table pointer");
  const HostSchedule* hs = get_schedule(model, dim);
  if (!hs) return fail(KGE_ERR_UNSUPPORTED, "kge_pack_table: unsupported dim");
  DeviceScope device_scope(ent0);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  int32_t* d_inv = nullptr;   // a stream-ordered allocation, freed on the same stream
  KGE_CUDA_TRY(cudaMallocAsync(reinterpret_cast<void**>(&d_inv), (size_t)dim * sizeof(int32_t), st),
               "pack_table: cudaMallocAsync");
  cudaError_t e = cudaMemcpyAsync(d_inv, hs->inv_perm.data(), (size_t)dim * sizeof(int32_t),
                                  cudaMemcpyHostToDevice, st);
  if (e == cudaSuccess)
    e = kge::launch_pack_table(ent0, ent1, planes, n_rows, dim, d_inv, packed, st);
  cudaError_t e2 = cudaFreeAsync(d_inv, st);
  if (e != cudaSuccess) return fail_cuda(e, "pack_table");
  if (e2 != cudaSuccess) return fail_cuda(e2, "pack_table: cudaFreeAsync");
  return KGE_OK;
}

int kge_gather_rows(int model, const float* ent0, const float* ent1, int64_t ent_lo,
                    int64_t n_rows, int dim, const int64_t* idx, int64_t n, float* out,
                    void* stream) {
  const int planes = kge_cand_planes(model);
  if (planes == 0) return fail(KGE_ERR_ARG, "kge_gather_rows: unknown model");
  if (n == 0) return KGE_OK;
  if (!ent0 || !idx || !out || (planes >= 2 && !ent1))
    return fail(KGE_ERR_ARG, "kge_gather_rows: null pointer");
  DeviceScope device_scope(ent0);
  KGE_CUDA_TRY(kge::launch_gather_rows(ent0, ent1, planes, ent_lo, n_rows, dim, idx, n, out,
                                       static_cast<cudaStream_t>(stream)),
               "gather_rows");
  return KGE_OK;
}

size_t kge_rank_workspace_bytes(int model, int side, int dim, int64_t n, int64_t n_rows, int flags) {
  const int el = kge::elem_kind_for(model, side);
  if (el < 0 || dim < 1 || n < 0) return 0;
  return carve(nullptr, kge::elem_qw(el), dim, n, el, n_rows, flags).bytes;
}

size_t kge_tc_packed_bytes(int model, int64_t n_rows, int dim) {
  const int el = kge::elem_kind_for(model, KGE_SIDE_TAIL);
  if (el < 0 || !tc_supported(el) || n_rows <= 0 || dim < 1) return 0;
  const int n_kb = kge::tc::n_kblocks(tc_k_total(el, dim));
  return TcImageLayout(n_rows, n_kb).total;
}

int kge_tc_configure(int bk, int resident, int ct_group, int max_ctas, int fp16) {
  kge::tc::configure(bk, resident, ct_group, max_ctas, fp16);
  return KGE_OK;
}

int kge_tc_layout_id(void) { return kge::tc::bk() * 2 + (kge::tc::fp16() ? 1 : 0); }

int kge_tc_bound_constants(int model, int dim, float* gamma, float* gamma2, float* gamma_p, int* fp16) {
  const int el = kge::elem_kind_for(model, KGE_SIDE_TAIL);
  if (el < 0 || !tc_supported(el)) return fail(KGE_ERR_UNSUPPORTED, "kge_tc_bound_constants: model has no tensor-core path");
  const HostSchedule* hs = get_schedule(model, dim);
  if (!hs) return fail(KGE_ERR_UNSUPPORTED, "kge_tc_bound_constants: unsupported dim");
  const int depth = kge::schedule_depth(hs->s);
  if (gamma) *gamma = kge::tc::tc_gamma(tc_k_total(el, dim), depth, tc_is_l2(el), kge::tc::fp16());
  if (gamma2) *gamma2 = kge::tc::tc_gamma2(depth);
  if (gamma_p) *gamma_p = kge::tc::tc_gamma_p();
  if (fp16) *fp16 = kge::tc::fp16() ? 1 : 0;
  return KGE_OK;
}

int kge_tc_pack_table(int model, const float* ent0, const float* ent1, int64_t n_rows, int dim,
                      void* tc_packed, void* stream) {
  return kge_tc_pack_table_cached(model, ent0, ent1, n_rows, dim, tc_packed, nullptr, stream);
}

int kge_tc_pack_table_cached(int model, const float* ent0, const float* ent1, int64_t n_rows, int dim,
                             void* tc_packed, uint64_t* guard, void* stream) {
  const int el = kge::elem_kind_for(model, KGE_SIDE_TAIL);
  if (el < 0 || !tc_supported(el)) return fail(KGE_ERR_UNSUPPORTED, "kge_tc_pack_table: model has no tensor-core path");
  if (n_rows <= 0) return KGE_OK;
  if (!ent0 || !tc_packed || (kge::elem_cw(el) >= 2 && !ent1))
    return fail(KGE_ERR_ARG, "kge_tc_pack_table: null pointer");
  // an image no scan could read (kge_rank_side rejects the same dims)
  if (!get_schedule(model, dim)) return fail(KGE_ERR_UNSUPPORTED, "kge_tc_pack_table: unsupported dim");
  DeviceScope device_scope(ent0);
  const int k_total = tc_k_total(el, dim);
  const int n_kb = kge::tc::n_kblocks(k_total);
  const TcImage<unsigned char> b(static_cast<unsigned char*>(tc_packed), n_rows, n_kb);
  KGE_CUDA_TRY(kge::tc::launch_pack_b(ent0, ent1, n_rows, dim, k_total, n_kb, tc_is_l2(el), b.bpack, b.cbound,
                                      b.cnorm2, b.cprefix, b.cbmax32, b.cpmax32, b.meta,
                                      reinterpret_cast<unsigned long long*>(guard),
                                      static_cast<cudaStream_t>(stream)),
               "tc pack table");
  return KGE_OK;
}

int kge_rank_side(const kge_rank_args_t* a) {
  QueryCall<kge_rank_args_t> q{"kge_rank_side", a};
  if (!a) return q.error(KGE_ERR_ARG, "null args");
  if (int rc = q.lookup_kind()) return rc;
  if (a->n == 0) return KGE_OK;
  if (a->n < 0 || a->n_rows < 0 || a->dim < 1) return q.error(KGE_ERR_ARG, "bad sizes");
  const int el = q.el;
  const bool rel_side = a->side == KGE_SIDE_REL;
  if (int rc = q.check_tables(a->ent0 && a->raw_count, kge::elem_cw(el) >= 2 && !a->ent1)) return rc;
  if (rel_side && !a->true_rows && !a->true_score_in)
    return q.error(KGE_ERR_ARG, "true_rows required for KGE_SIDE_REL");
  if (a->filt_offs && (!a->filt_ids || !a->filt_sub) && a->n_filt > 0)
    return q.error(KGE_ERR_ARG, "filter arrays incomplete");
  if (int rc = q.lookup_schedule()) return rc;
  const bool use_tc = (a->flags & KGE_FLAG_TENSOR_CORE) && tc_supported(el) && a->n_rows > 0;
  if (use_tc && !a->tc_packed) return q.error(KGE_ERR_ARG, "tc_packed required with KGE_FLAG_TENSOR_CORE");
  if (!use_tc && !a->packed) return q.error(KGE_ERR_ARG, "packed table required (scalar scan)");
  const bool use_approx = !use_tc && (a->flags & KGE_FLAG_APPROX_SCAN) && approx_supported(el) && a->n_rows > 0;
  const int qw = kge::elem_qw(el);
  const Workspace w = carve(a->workspace, qw, a->dim, a->n, el, a->n_rows,
                            use_tc ? KGE_FLAG_TENSOR_CORE : (use_approx ? KGE_FLAG_APPROX_SCAN : 0));
  if (int rc = q.prepare(a->ent0, w, w.bytes, !use_tc)) return rc;
  cudaStream_t st = q.stream();
  const HostSchedule* hs = q.hs;
  const bool casc = hs->s.has_cascade;

  // true scores: the true entity's row is the gathered tail (tail side) / head (head side) row
  const int64_t n_qt = (a->n + kge::TILE_Q - 1) / kge::TILE_Q;
  const float nan_v = __builtin_nanf("");
  KGE_CUDA_TRY(kge::launch_fill_f32(w.s_true + a->n, nan_v, n_qt * kge::TILE_Q - a->n, st),
               "fill s_true pad");
  const float* true_rows = a->true_rows ? a->true_rows : (a->side == KGE_SIDE_TAIL ? a->trows : a->hrows);
  if (a->true_score_in)
    KGE_CUDA_TRY(cudaMemcpyAsync(w.s_true, a->true_score_in, (size_t)a->n * sizeof(float),
                                 cudaMemcpyDeviceToDevice, st),
                 "copy true_score_in");
  else
    KGE_CUDA_TRY(kge::launch_true_scores(el, casc, a->dim, a->n, w.qplain, true_rows, w.perm, w.code,
                                         w.s_true, st),
                 "true_scores");
  if (a->true_score)
    KGE_CUDA_TRY(cudaMemcpyAsync(a->true_score, w.s_true, (size_t)a->n * sizeof(float),
                                 cudaMemcpyDeviceToDevice, st),
                 "copy true_score");
  if (a->n_rows == 0) return KGE_OK;

  if (use_tc) {
    // tensor-core bound-and-refine: approximate scores decide all but the near-tie band,
    // which is re-scored exactly (same device functions as the scalar scan)
    const int k_total = tc_k_total(el, a->dim);
    const int n_kb = kge::tc::n_kblocks(k_total);
    const bool l2 = tc_is_l2(el);
    const TcImage<const unsigned char> b(static_cast<const unsigned char*>(a->tc_packed), a->n_rows, n_kb);
    KGE_CUDA_TRY(kge::tc::launch_pack_a(w.qplain, qw, a->n, a->dim, k_total, n_kb,
                                        el == kge::EL_L2_HEAD ? 1 : 0, l2, w.apack, w.qbound, w.qnorm2, w.qprefix,
                                        w.meta_a, b.meta, st),
                 "tc pack queries");
    if (kge::tc::scan_grid_size(a->n, a->n_rows, n_kb) <= 0)
      return fail(KGE_ERR_CUDA, "kge_rank_side: cannot size the tensor-core grid");
    kge::tc::TcScanParams tp;
    tp.meta_a = w.meta_a; tp.meta_b = b.meta;
    tp.apack = w.apack; tp.bpack = b.bpack; tp.s_true = w.s_true;
    tp.qbound = w.qbound; tp.qnorm2 = w.qnorm2;
    tp.cbound = b.cbound; tp.cnorm2 = b.cnorm2; tp.cprefix = b.cprefix;
    tp.cbmax32 = b.cbmax32; tp.cpmax32 = b.cpmax32; tp.qprefix = w.qprefix;
    tp.gamma_p = kge::tc::tc_gamma_p();
    tp.counts = a->raw_count; tp.amb_count = w.amb_count; tp.amb_pairs = w.amb_pairs;
    tp.dump = a->tc_dump;
    const int ref_depth = kge::schedule_depth(hs->s);
    tp.gamma = kge::tc::tc_gamma(k_total, ref_depth, l2, kge::tc::fp16()); tp.gamma2 = kge::tc::tc_gamma2(ref_depth);
    tp.l2 = l2 ? 1 : 0;
    tp.n_kb = n_kb; tp.k_total = k_total;
    tp.n_q = a->n; tp.n_rows = a->n_rows;
    tp.n_qt = (a->n + kge::tc::TC_BM - 1) / kge::tc::TC_BM; tp.n_ct = (a->n_rows + kge::tc::TC_BN - 1) / kge::tc::TC_BN;
    if (int rc = refine(true, a, el, w, st, [&](unsigned long long region_cap) {
          tp.amb_cap = region_cap;
          return kge::tc::launch_tc_scan(tp, st);
        }))
      return rc;
  } else {
    kge::ScanParams p = scan_params(a->packed, w.qpacked, w.s_true, hs, a->dim, a->n, a->n_rows);
    p.counts = a->raw_count;
    if (use_approx) {
      // RotatE bound-and-refine: |s~ - s_ATen| <= rel_eps |s~| (all terms >= 0).  Per element the
      // exact path is within 4 u and the approximate one within 3 u + 2^-21 (sqrt.approx) of the
      // real modulus; the sums add depth * u each: ATen's cascade (schedule_depth) for the exact
      // path, 32 per stage + one per stage for the approximate one.
      const int depth_a = 32 + (a->dim + 31) / 32, depth_e = kge::schedule_depth(hs->s);
      p.amb_count = w.amb_count; p.amb_pairs = w.amb_pairs;
      p.rel_eps = (float)((depth_a + depth_e + 4 + 11 + 8) * 0x1p-24 * 1.001);
      p.abs_eps = (float)(a->dim * 1.1e-19);
      if (int rc = refine(false, a, el, w, st, [&](unsigned long long region_cap) {
            p.amb_cap = region_cap;
            return kge::launch_scan(el, casc, p, st, true);
          }))
        return rc;
    } else {
      KGE_CUDA_TRY(timed_scan(el, casc, p, st), "rank scan");
    }
  }
  if (a->filt_offs && a->n_filt > 0) KGE_CUDA_TRY(launch_filter_pass(a, el, casc, w, st), "filter pass");
  return KGE_OK;
}

int kge_filter_side(const kge_rank_args_t* a) {
  if (!a) return fail(KGE_ERR_ARG, "kge_filter_side: null args");
  const int el = kge::elem_kind_for(a->model, a->side);
  if (el < 0) return fail(KGE_ERR_ARG, "kge_filter_side: unknown model/side");
  if (a->n == 0 || a->n_filt == 0 || a->n_rows == 0) return KGE_OK;
  if (!a->ent0 || !a->filt_offs || !a->filt_ids || !a->filt_sub || !a->workspace)
    return fail(KGE_ERR_ARG, "kge_filter_side: null pointer");
  if (kge::elem_cw(el) >= 2 && !a->ent1) return fail(KGE_ERR_ARG, "kge_filter_side: ent1 required");
  const HostSchedule* hs = get_schedule(a->model, a->dim);
  if (!hs) return fail(KGE_ERR_UNSUPPORTED, "kge_filter_side: unsupported dim");
  DeviceScope device_scope(a->ent0);
  Workspace w = carve(a->workspace, kge::elem_qw(el), a->dim, a->n);  // leading part only
  if (w.bytes > a->workspace_bytes) return fail(KGE_ERR_ARG, "kge_filter_side: workspace too small");
  KGE_CUDA_TRY(launch_filter_pass(a, el, hs->s.has_cascade, w, static_cast<cudaStream_t>(a->stream)), "filter pass");
  return KGE_OK;
}

int kge_finalize_ranks(const int32_t* raw_count, const int32_t* filt_sub, int64_t n,
                       int64_t* ranks, int64_t* filt_ranks, void* stream) {
  if (n == 0) return KGE_OK;
  if (!raw_count || !filt_sub || !ranks || !filt_ranks)
    return fail(KGE_ERR_ARG, "kge_finalize_ranks: null pointer");
  DeviceScope device_scope(raw_count);
  KGE_CUDA_TRY(kge::launch_finalize(raw_count, filt_sub, n, ranks, filt_ranks,
                                    static_cast<cudaStream_t>(stream)),
               "finalize");
  return KGE_OK;
}

int kge_score_all(const kge_score_all_args_t* a) {
  QueryCall<kge_score_all_args_t> q{"kge_score_all", a};
  if (!a) return q.error(KGE_ERR_ARG, "null args");
  if (int rc = q.lookup_kind()) return rc;
  if (a->n == 0 || a->n_rows == 0) return KGE_OK;
  if (int rc = q.check_tables(a->packed && a->scores)) return rc;
  if (int rc = q.lookup_schedule()) return rc;
  const Workspace w = carve(a->workspace, kge::elem_qw(q.el), a->dim, a->n);
  if (int rc = q.prepare(a->packed, w, w.bytes)) return rc;
  cudaStream_t st = q.stream();
  const int64_t n_qt = (a->n + kge::TILE_Q - 1) / kge::TILE_Q;
  KGE_CUDA_TRY(kge::launch_fill_f32(w.s_true, 0.f, n_qt * kge::TILE_Q, st), "fill s_true");
  kge::ScanParams p = scan_params(a->packed, w.qpacked, w.s_true, q.hs, a->dim, a->n, a->n_rows);
  p.scores = a->scores;
  KGE_CUDA_TRY(timed_scan(q.el, q.hs->s.has_cascade, p, st), "score scan");
  return KGE_OK;
}

// ------------------------------------ top-k inference ------------------------------------
namespace {
// candidate rows scanned per collect pass: the per-query lists of one pass hold at most this many
// entries each (8 bytes), bounded to 256 MB in total, a multiple of the scan's candidate tile
int64_t topk_chunk_rows(int64_t n, int64_t n_rows) {
  const int64_t budget = (int64_t)256 << 20;
  int64_t rows = budget / (8 * (n > 0 ? n : 1));
  rows = rows / kge::TILE_C * kge::TILE_C;
  if (rows < kge::TILE_C) rows = kge::TILE_C;
  const int64_t all = (n_rows + kge::TILE_C - 1) / kge::TILE_C * kge::TILE_C;
  return rows < all ? rows : all;
}
struct TopkWorkspace {
  Workspace w;
  float* thr;
  unsigned* col_count;
  int2* col_buf;
  unsigned long long* best;
  int64_t chunk_rows;
  size_t bytes;
};
TopkWorkspace carve_topk(void* base, int qw, int dim, int64_t n, int64_t n_rows, int k) {
  TopkWorkspace t;
  t.w = carve(base, qw, dim, n);
  Carver c{base, t.w.bytes};
  const int64_t n_qt = (n + kge::TILE_Q - 1) / kge::TILE_Q;
  t.chunk_rows = topk_chunk_rows(n, n_rows);
  t.thr = c.take<float>((size_t)n_qt * kge::TILE_Q * sizeof(float));
  t.col_count = c.take<unsigned>((size_t)n * sizeof(unsigned));
  t.col_buf = c.take<int2>((size_t)n * t.chunk_rows * sizeof(int2));
  t.best = c.take<unsigned long long>((size_t)n * k * sizeof(unsigned long long));
  t.bytes = c.off;
  return t;
}
}  // namespace

size_t kge_topk_workspace_bytes(int model, int side, int dim, int64_t n, int64_t n_rows, int k) {
  const int el = kge::elem_kind_for(model, side);
  if (el < 0 || dim < 1 || n < 0 || n_rows < 0 || k < 1 || k > kge::TOPK_MAX_K) return 0;
  return carve_topk(nullptr, kge::elem_qw(el), dim, n, n_rows, k).bytes;
}

int kge_topk_side(const kge_topk_args_t* a) {
  QueryCall<kge_topk_args_t> q{"kge_topk_side", a};
  if (!a) return q.error(KGE_ERR_ARG, "null args");
  if (int rc = q.lookup_kind()) return rc;
  if (a->k < 1 || a->k > kge::TOPK_MAX_K) return q.error(KGE_ERR_ARG, "k must be in [1, 1024]");
  if (a->n < 0 || a->n_rows < 0 || a->dim < 1) return q.error(KGE_ERR_ARG, "bad sizes");
  if ((int64_t)a->k > a->n_rows) return q.error(KGE_ERR_ARG, "k exceeds the number of candidates");
  // candidate ids travel as int32 through the collect lists and the 64-bit keys
  if (a->ent_lo < 0 || a->ent_lo + a->n_rows > (int64_t)INT32_MAX)
    return q.error(KGE_ERR_ARG, "ent_lo + n_rows must lie in [0, 2^31 - 1]");
  if (a->n == 0) return KGE_OK;
  if (int rc = q.check_tables(a->packed && a->pred && a->scores)) return rc;
  if (a->mask_offs && !a->mask_ids) return q.error(KGE_ERR_ARG, "mask arrays incomplete");
  if (int rc = q.lookup_schedule()) return rc;
  const int cw = kge::elem_cw(q.el);
  const TopkWorkspace t = carve_topk(a->workspace, kge::elem_qw(q.el), a->dim, a->n, a->n_rows, a->k);
  if (int rc = q.prepare(a->packed, t.w, t.bytes)) return rc;
  cudaStream_t st = q.stream();
  const int64_t n_qt = (a->n + kge::TILE_Q - 1) / kge::TILE_Q;
  KGE_CUDA_TRY(kge::launch_fill_f32(t.thr, -__builtin_inff(), n_qt * kge::TILE_Q, st), "topk: thresholds");
  KGE_CUDA_TRY(cudaMemsetAsync(t.best, 0, (size_t)a->n * a->k * sizeof(unsigned long long), st), "topk: reset lists");
  for (int64_t c0 = 0; c0 < a->n_rows; c0 += t.chunk_rows) {
    const int64_t rows = a->n_rows - c0 < t.chunk_rows ? a->n_rows - c0 : t.chunk_rows;
    const bool first = c0 == 0;   // thresholds are -inf: every candidate is collected, slot = row
    if (!first) KGE_CUDA_TRY(cudaMemsetAsync(t.col_count, 0, (size_t)a->n * sizeof(unsigned), st), "topk: reset counts");
    kge::ScanParams p = scan_params(a->packed + (size_t)(c0 / kge::TILE_C) * a->dim * cw * kge::TILE_C, t.w.qpacked,
                                    t.thr, q.hs, a->dim, a->n, rows);
    p.col_buf = t.col_buf; p.col_count = t.col_count; p.col_cap = (unsigned long long)t.chunk_rows;
    p.col_id_base = a->ent_lo + c0; p.col_dense = first ? 1 : 0;
    KGE_CUDA_TRY(timed_scan(q.el, q.hs->s.has_cascade, p, st), "topk: collect scan");
    KGE_CUDA_TRY(kge::launch_topk_merge(t.best, a->k, t.col_buf, t.col_count, (unsigned long long)t.chunk_rows,
                                        first ? rows : -1, a->mask_offs, a->mask_ids, t.thr, a->n, st),
                 "topk: merge");
  }
  KGE_CUDA_TRY(kge::launch_topk_finish(t.best, a->k, a->n, a->pred, a->scores, st), "topk: finish");
  return KGE_OK;
}

int kge_topk_merge(const int64_t* pred_in, const float* scores_in, int n_lists, int64_t n, int k_in, int k,
                   int64_t* pred, float* scores, void* stream) {
  if (n_lists < 1 || n_lists > kge::TOPK_MAX_LISTS)
    return fail(KGE_ERR_ARG, "kge_topk_merge: n_lists must be in [1, 64]");
  if (k < 1 || k > kge::TOPK_MAX_K) return fail(KGE_ERR_ARG, "kge_topk_merge: k must be in [1, 1024]");
  if (k_in < 1 || k_in > kge::TOPK_MAX_K) return fail(KGE_ERR_ARG, "kge_topk_merge: k_in must be in [1, 1024]");
  if (n < 0) return fail(KGE_ERR_ARG, "kge_topk_merge: bad sizes");
  if (n == 0) return KGE_OK;
  if (!pred_in || !scores_in || !pred || !scores) return fail(KGE_ERR_ARG, "kge_topk_merge: null pointer");
  DeviceScope device_scope(pred);
  KGE_CUDA_TRY(kge::launch_topk_lists_merge(pred_in, scores_in, n_lists, n, k_in, k, pred, scores,
                                            static_cast<cudaStream_t>(stream)),
               "topk_merge");
  return KGE_OK;
}

// ------------------------------------ dense side paths ------------------------------------
int kge_rescal_rel_scores(const float* hrows, const float* trows, const float* rel_mat, int dim, int64_t n,
                          int64_t n_rel, float* scores, void* stream) {
  if (n == 0 || n_rel == 0) return KGE_OK;
  if (n < 0 || n_rel < 0 || dim < 1 || !hrows || !trows || !rel_mat || !scores)
    return fail(KGE_ERR_ARG, "kge_rescal_rel_scores: bad argument");
  if (dim > 2048) return fail(KGE_ERR_UNSUPPORTED, "kge_rescal_rel_scores: dim > 2048");
  DeviceScope device_scope(scores);
  KGE_CUDA_TRY(kge::launch_rescal_rel_scores(hrows, trows, rel_mat, dim, n, n_rel, scores,
                                             static_cast<cudaStream_t>(stream)),
               "rescal_rel_scores");
  return KGE_OK;
}

int kge_transh_rel_scores(const float* hrows, const float* trows, const float* rel, const float* norm_vect,
                          int dim, int64_t n, int64_t n_rel, float* scores, void* stream) {
  if (n == 0 || n_rel == 0) return KGE_OK;
  if (n < 0 || n_rel < 0 || dim < 1 || !hrows || !trows || !rel || !norm_vect || !scores)
    return fail(KGE_ERR_ARG, "kge_transh_rel_scores: bad argument");
  if (dim > kge::SCAN_MAX_DIM) return fail(KGE_ERR_UNSUPPORTED, "kge_transh_rel_scores: dim > 8192");
  DeviceScope device_scope(scores);
  KGE_CUDA_TRY(kge::launch_transh_rel_scores(hrows, trows, rel, norm_vect, dim, n, n_rel, scores,
                                             static_cast<cudaStream_t>(stream)),
               "transh_rel_scores");
  return KGE_OK;
}

int kge_transh_project(const float* ent, const float* norm_row, int64_t n_rows, int dim, float* out,
                       void* stream) {
  if (n_rows == 0) return KGE_OK;
  if (n_rows < 0 || dim < 1 || !ent || !norm_row || !out) return fail(KGE_ERR_ARG, "kge_transh_project: bad argument");
  if (dim > kge::SCAN_MAX_DIM) return fail(KGE_ERR_UNSUPPORTED, "kge_transh_project: dim > 8192");
  DeviceScope device_scope(out);
  KGE_CUDA_TRY(kge::launch_transh_project(ent, norm_row, n_rows, dim, out, static_cast<cudaStream_t>(stream)),
               "transh_project");
  return KGE_OK;
}

int kge_transd_entity_scalars(const float* ent, const float* ent_proj, int64_t n_rows, int ent_dim, float* s,
                              void* stream) {
  if (n_rows == 0) return KGE_OK;
  if (n_rows < 0 || ent_dim < 1 || !ent || !ent_proj || !s)
    return fail(KGE_ERR_ARG, "kge_transd_entity_scalars: bad argument");
  if (ent_dim > kge::SCAN_MAX_DIM) return fail(KGE_ERR_UNSUPPORTED, "kge_transd_entity_scalars: ent_dim > 8192");
  DeviceScope device_scope(s);
  KGE_CUDA_TRY(kge::launch_transd_entity_scalars(ent, ent_proj, n_rows, ent_dim, s, static_cast<cudaStream_t>(stream)),
               "transd_entity_scalars");
  return KGE_OK;
}

int kge_transd_project(const float* ent, int ent_dim, const float* s, const float* rel_proj_row, int64_t n_rows,
                       int rel_dim, float* out, void* stream) {
  if (n_rows == 0) return KGE_OK;
  if (n_rows < 0 || rel_dim < 1 || ent_dim < 1 || !ent || !s || !rel_proj_row || !out)
    return fail(KGE_ERR_ARG, "kge_transd_project: bad argument");
  if (rel_dim > ent_dim) return fail(KGE_ERR_ARG, "kge_transd_project: rel_dim > ent_dim");
  if (ent_dim > kge::SCAN_MAX_DIM) return fail(KGE_ERR_UNSUPPORTED, "kge_transd_project: ent_dim > 8192");
  DeviceScope device_scope(out);
  KGE_CUDA_TRY(kge::launch_transd_project(ent, ent_dim, s, rel_proj_row, n_rows, rel_dim, out,
                                          static_cast<cudaStream_t>(stream)),
               "transd_project");
  return KGE_OK;
}

int kge_transd_rel_scores(const float* hrows, const float* hs, const float* trows, const float* ts, const float* rel,
                          const float* rel_proj, int rel_dim, int64_t n, int64_t n_rel, float* scores, void* stream) {
  if (n == 0 || n_rel == 0) return KGE_OK;
  if (n < 0 || n_rel < 0 || rel_dim < 1 || !hrows || !hs || !trows || !ts || !rel || !rel_proj || !scores)
    return fail(KGE_ERR_ARG, "kge_transd_rel_scores: bad argument");
  if (rel_dim > kge::SCAN_MAX_DIM) return fail(KGE_ERR_UNSUPPORTED, "kge_transd_rel_scores: rel_dim > 8192");
  DeviceScope device_scope(scores);
  KGE_CUDA_TRY(kge::launch_transd_rel_scores(hrows, hs, trows, ts, rel, rel_proj, rel_dim, n, n_rel, scores,
                                             static_cast<cudaStream_t>(stream)),
               "transd_rel_scores");
  return KGE_OK;
}

int kge_rank_dense(const float* scores, int64_t n, int64_t n_cand, const int64_t* true_idx,
                   const float* true_score_in, const int64_t* filt_offs, const int64_t* filt_ids,
                   int32_t* raw_count, int32_t* filt_sub, float* true_score, void* stream) {
  if (n == 0) return KGE_OK;
  if (n < 0 || n_cand < 1 || !scores || !raw_count || (!true_idx && !true_score_in) || (filt_offs && (!filt_ids || !filt_sub)))
    return fail(KGE_ERR_ARG, "kge_rank_dense: bad argument");
  DeviceScope device_scope(scores);
  KGE_CUDA_TRY(kge::launch_rank_dense(scores, n, n_cand, true_idx, true_score_in, filt_offs, filt_ids, raw_count,
                                      filt_sub, true_score, static_cast<cudaStream_t>(stream)),
               "rank_dense");
  return KGE_OK;
}

size_t kge_topk_dense_workspace_bytes(int64_t n, int64_t n_cand, int k) {
  if (n < 0 || n_cand < 1 || k < 1 || k > kge::TOPK_MAX_K) return 0;
  return align_up((size_t)n * n_cand * sizeof(int2), 256) + align_up((size_t)n * k * sizeof(unsigned long long), 256) +
         align_up((size_t)n * sizeof(float), 256);
}

int kge_topk_dense(const float* scores, int64_t n, int64_t n_cand, int k, const int64_t* mask_offs,
                   const int64_t* mask_ids, int64_t* pred, float* out_scores, void* workspace,
                   size_t workspace_bytes, void* stream) {
  if (n == 0) return KGE_OK;
  if (n < 0 || n_cand < 1 || k < 1 || k > kge::TOPK_MAX_K || k > n_cand || !scores || !pred || !out_scores || !workspace)
    return fail(KGE_ERR_ARG, "kge_topk_dense: bad argument");
  if (kge_topk_dense_workspace_bytes(n, n_cand, k) > workspace_bytes)
    return fail(KGE_ERR_ARG, "kge_topk_dense: workspace too small");
  DeviceScope device_scope(scores);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  char* base = static_cast<char*>(workspace);
  int2* pairs = reinterpret_cast<int2*>(base);
  unsigned long long* best = reinterpret_cast<unsigned long long*>(base + align_up((size_t)n * n_cand * sizeof(int2), 256));
  float* thr = reinterpret_cast<float*>(reinterpret_cast<char*>(best) + align_up((size_t)n * k * sizeof(unsigned long long), 256));
  KGE_CUDA_TRY(cudaMemsetAsync(best, 0, (size_t)n * k * sizeof(unsigned long long), st), "topk_dense: reset");
  KGE_CUDA_TRY(kge::launch_dense_to_pairs(scores, n, n_cand, pairs, st), "topk_dense: pairs");
  KGE_CUDA_TRY(kge::launch_topk_merge(best, k, pairs, nullptr, (unsigned long long)n_cand, n_cand, mask_offs, mask_ids,
                                      thr, n, st),
               "topk_dense: merge");
  KGE_CUDA_TRY(kge::launch_topk_finish(best, k, n, pred, out_scores, st), "topk_dense: finish");
  return KGE_OK;
}

int kge_cooccurrence(const int64_t* left_keys, const int64_t* left_offs, const int64_t* left_pairs, int64_t n_left,
                     const int64_t* right_keys, const int64_t* right_offs, const int64_t* right_pairs, int64_t n_right,
                     int64_t n_ent, int64_t n_rel, int flip, int upper, uint64_t* counts, void* stream) {
  if (n_left == 0 || n_right == 0) return KGE_OK;
  if (n_left < 0 || n_right < 0 || n_ent < 1 || n_rel < 1)
    return fail(KGE_ERR_ARG, "kge_cooccurrence", "bad sizes");
  if (!left_keys || !left_offs || !left_pairs || !right_keys || !right_offs || !right_pairs || !counts)
    return fail(KGE_ERR_ARG, "kge_cooccurrence", "null pointer");
  DeviceScope device_scope(counts);
  KGE_CUDA_TRY(kge::launch_cooccurrence(left_keys, left_offs, left_pairs, n_left, right_keys, right_offs, right_pairs,
                                        n_right, n_ent, n_rel, flip != 0, upper != 0,
                                        reinterpret_cast<unsigned long long*>(counts),
                                        static_cast<cudaStream_t>(stream)),
               "cooccurrence");
  return KGE_OK;
}

// ------------------------------------ training side ------------------------------------
namespace {
bool tables_ok(const kge_tables_t* tb) {
  if (!tb || !tb->ent0 || !tb->rel0 || tb->dim < 1) return false;
  if (tb->model < KGE_TRANSE_L1 || tb->model > KGE_ANALOGY) return false;
  if (model_needs_rel1(tb->model) && (!tb->ent1 || !tb->rel1)) return false;
  return true;
}
bool grads_ok(const kge_tables_t* tb, const kge_grads_t* g) {
  if (!g || !g->ent0 || !g->rel0) return false;
  if (model_needs_rel1(tb->model) && (!g->ent1 || !g->rel1)) return false;
  return true;
}
kge::TrainTables to_tables(const kge_tables_t* tb) {
  return kge::TrainTables{tb->ent0, tb->ent1, tb->rel0, tb->rel1};
}
kge::TrainGrads to_grads(const kge_grads_t* g) { return kge::TrainGrads{g->ent0, g->ent1, g->rel0, g->rel1}; }
kge::MarginStepParams to_step(const kge_margin_step_args_t* a) {
  kge::MarginStepParams p;
  p.model = a->tb.model; p.dim = a->tb.dim; p.n_neg = a->n_neg; p.margin = a->margin;
  p.b = a->b; p.n_ent = a->n_ent; p.tb = to_tables(&a->tb);
  p.h = a->h; p.t = a->t; p.r = a->r; p.nh = a->nh; p.nt = a->nt; p.probs = a->bern_probs;
  p.seed = a->seed; p.offset = a->offset; p.loss = a->loss; p.pos_out = a->pos_out;
  p.neg_out = a->neg_out; p.nh_out = a->nh_out; p.nt_out = a->nt_out;
  p.ent_lo = a->ent_lo; p.n_rows = a->n_rows; p.hrows = a->hrows; p.trows = a->trows;
  p.grad_hrows = a->grad_hrows; p.grad_trows = a->grad_trows;
  p.loss_kind = a->loss_kind;
  p.n_rel = 0; p.rel_share = 1.f; p.nr = nullptr; p.nr_out = nullptr;   // the entity step
  return p;
}
kge::PosCSR to_pos_csr(const kge_pos_step_args_t* a) {
  return kge::PosCSR{a->head_offs, a->head_ents, a->tail_offs, a->tail_ents};
}
kge::MarginStepParams to_rel_step(const kge_rel_step_args_t* a) {
  kge::MarginStepParams p = to_step(&a->base);
  p.n_rel = a->n_rel; p.rel_share = a->rel_share; p.nr = a->nr; p.nr_out = a->nr_out;
  return p;
}
// n_rel >= 2 unless every negative replaces an entity; a NaN rel_share fails the range test
bool rel_draw_ok(int64_t n_rel, float rel_share) {
  return rel_share >= 0.f && rel_share <= 1.f && n_rel >= 1 && (n_rel >= 2 || rel_share >= 1.f);
}
// A shard that holds no rows (n_rows = 0) may pass no entity planes.
bool step_tables_ok(const kge_margin_step_args_t* a) {
  if (tables_ok(&a->tb)) return true;
  if (!a->hrows || a->n_rows != 0) return false;
  kge_tables_t tb = a->tb;
  tb.ent0 = a->hrows;
  tb.ent1 = a->hrows;
  return tables_ok(&tb);
}
bool step_grads_ok(const kge_margin_step_args_t* a, const kge_grads_t* g) {
  if (grads_ok(&a->tb, g)) return true;
  if (!g || !a->hrows || a->n_rows != 0) return false;
  kge_grads_t gg = *g;
  gg.ent0 = gg.ent1 = a->grad_hrows;
  return grads_ok(&a->tb, &gg);
}
bool step_ok(const kge_margin_step_args_t* a) {
  if (!a || !step_tables_ok(a) || a->b < 0 || a->n_neg < 1 || !a->loss) return false;
  if (a->b > 0 && (!a->h || !a->t || !a->r)) return false;
  if ((a->nh == nullptr) != (a->nt == nullptr)) return false;
  if (!a->nh && !a->bern_probs) return false;
  if ((a->nh_out == nullptr) != (a->nt_out == nullptr)) return false;
  if (a->loss_kind != KGE_LOSS_MARGIN && a->loss_kind != KGE_LOSS_LOGISTIC && a->loss_kind != KGE_LOSS_BCE)
    return false;
  if (a->hrows) {   // entity-sharded: Philox draws only, no per-negative outputs
    if (!a->trows || a->nh || a->pos_out || a->neg_out || a->nh_out) return false;
    if (a->ent_lo < 0 || a->n_rows < 0 || a->ent_lo + a->n_rows > a->n_ent) return false;
  }
  return true;
}
bool shard_grads_ok(const kge_margin_step_args_t* a) {
  return !a->hrows || (a->grad_hrows && a->grad_trows);
}
bool rel_step_ok(const kge_rel_step_args_t* a) {
  if (!a || !step_ok(&a->base) || !rel_draw_ok(a->n_rel, a->rel_share)) return false;
  if ((a->nr == nullptr) != (a->base.nh == nullptr)) return false;
  if (a->base.hrows && a->nr_out) return false;   // sharded: no per-negative outputs
  return true;
}
// An ents array may be NULL only when offs[n_rel] == offs[0]: read from the device, on the step's stream, in
// that case alone (an empty side), so a well-formed step never waits for the device here.
bool pos_side_ok(const int64_t* offs, const int64_t* ents, int64_t n_rel, void* stream) {
  if (ents) return true;
  int64_t ends[2] = {0, 1};
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (cudaMemcpyAsync(&ends[0], offs, sizeof(int64_t), cudaMemcpyDeviceToHost, st) != cudaSuccess ||
      cudaMemcpyAsync(&ends[1], offs + n_rel, sizeof(int64_t), cudaMemcpyDeviceToHost, st) != cudaSuccess ||
      cudaStreamSynchronize(st) != cudaSuccess) {
    cudaGetLastError();   // a bad offs pointer is an argument error, not a sticky one
    return false;
  }
  return ends[0] == ends[1];
}
bool pos_step_ok(const kge_pos_step_args_t* a) {
  if (!a || !step_ok(&a->base) || a->n_rel < 1 || !a->head_offs || !a->tail_offs) return false;
  if (a->base.nh) return false;   // caller negatives would make the draw meaningless
  return pos_side_ok(a->head_offs, a->head_ents, a->n_rel, a->base.stream) &&
         pos_side_ok(a->tail_offs, a->tail_ents, a->n_rel, a->base.stream);
}
}  // namespace

int kge_score_triples_fwd(const kge_tables_t* tb, const int64_t* h, const int64_t* t,
                          const int64_t* r, int64_t n, float* scores, void* stream) {
  if (!tables_ok(tb)) return fail(KGE_ERR_ARG, "kge_score_triples_fwd: bad tables");
  if (n == 0) return KGE_OK;
  if (n < 0 || !h || !t || !r || !scores) return fail(KGE_ERR_ARG, "kge_score_triples_fwd: null pointer");
  DeviceScope device_scope(tb->ent0);
  KGE_CUDA_TRY(kge::launch_score_triples_fwd(tb->model, tb->dim, to_tables(tb), h, t, r, n, scores,
                                             static_cast<cudaStream_t>(stream)),
               "score_triples_fwd");
  return KGE_OK;
}

int kge_score_triples_bwd(const kge_tables_t* tb, const kge_grads_t* g, const int64_t* h,
                          const int64_t* t, const int64_t* r, int64_t n, const float* grad_scores,
                          void* stream) {
  if (!tables_ok(tb) || !grads_ok(tb, g)) return fail(KGE_ERR_ARG, "kge_score_triples_bwd: bad tables");
  if (n == 0) return KGE_OK;
  if (n < 0 || !h || !t || !r || !grad_scores)
    return fail(KGE_ERR_ARG, "kge_score_triples_bwd: null pointer");
  DeviceScope device_scope(tb->ent0);
  KGE_CUDA_TRY(kge::launch_score_triples_bwd(tb->model, tb->dim, to_tables(tb), to_grads(g), h, t, r, n,
                                             grad_scores, static_cast<cudaStream_t>(stream)),
               "score_triples_bwd");
  return KGE_OK;
}

int kge_transh_score_triples_fwd(const float* ent, const float* rel, const float* norm_vect, int dim,
                                 const int64_t* h, const int64_t* t, const int64_t* r, int64_t n, float* scores,
                                 void* stream) {
  if (n == 0) return KGE_OK;
  if (n < 0 || dim < 1 || !ent || !rel || !norm_vect || !h || !t || !r || !scores)
    return fail(KGE_ERR_ARG, "kge_transh_score_triples_fwd: bad argument");
  DeviceScope device_scope(ent);
  KGE_CUDA_TRY(kge::launch_transh_score_fwd(ent, rel, norm_vect, dim, h, t, r, n, scores,
                                            static_cast<cudaStream_t>(stream)),
               "transh_score_triples_fwd");
  return KGE_OK;
}

int kge_transh_score_triples_bwd(const float* ent, const float* rel, const float* norm_vect, float* grad_ent,
                                 float* grad_rel, float* grad_norm_vect, int dim, const int64_t* h,
                                 const int64_t* t, const int64_t* r, int64_t n, const float* grad_scores,
                                 void* stream) {
  if (n == 0) return KGE_OK;
  if (n < 0 || dim < 1 || !ent || !rel || !norm_vect || !grad_ent || !grad_rel || !grad_norm_vect || !h || !t ||
      !r || !grad_scores)
    return fail(KGE_ERR_ARG, "kge_transh_score_triples_bwd: bad argument");
  DeviceScope device_scope(ent);
  KGE_CUDA_TRY(kge::launch_transh_score_bwd(ent, rel, norm_vect, grad_ent, grad_rel, grad_norm_vect, dim, h, t, r,
                                            n, grad_scores, static_cast<cudaStream_t>(stream)),
               "transh_score_triples_bwd");
  return KGE_OK;
}

// TransD's widths: rel_dim <= ent_dim (the reference's projection fails otherwise), both within SCAN_MAX_DIM
static int transd_widths(int ent_dim, int rel_dim, const char* fn) {
  if (ent_dim < 1 || rel_dim < 1 || rel_dim > ent_dim) return fail(KGE_ERR_ARG, fn, "need 1 <= rel_dim <= ent_dim");
  if (ent_dim > kge::SCAN_MAX_DIM) return fail(KGE_ERR_UNSUPPORTED, fn, "ent_dim > 8192");
  return KGE_OK;
}

int kge_transd_score_triples_fwd(const float* ent, const float* rel, const float* ent_proj, const float* rel_proj,
                                 int ent_dim, int rel_dim, const int64_t* h, const int64_t* t, const int64_t* r,
                                 int64_t n, float* scores, void* stream) {
  if (n == 0) return KGE_OK;
  if (n < 0 || !ent || !rel || !ent_proj || !rel_proj || !h || !t || !r || !scores)
    return fail(KGE_ERR_ARG, "kge_transd_score_triples_fwd: bad argument");
  if (int e = transd_widths(ent_dim, rel_dim, "kge_transd_score_triples_fwd")) return e;
  DeviceScope device_scope(ent);
  KGE_CUDA_TRY(kge::launch_transd_score_fwd(ent, rel, ent_proj, rel_proj, ent_dim, rel_dim, h, t, r, n, scores,
                                            static_cast<cudaStream_t>(stream)),
               "transd_score_triples_fwd");
  return KGE_OK;
}

int kge_transd_score_triples_bwd(const float* ent, const float* rel, const float* ent_proj, const float* rel_proj,
                                 float* grad_ent, float* grad_rel, float* grad_ent_proj, float* grad_rel_proj,
                                 int ent_dim, int rel_dim, const int64_t* h, const int64_t* t, const int64_t* r,
                                 int64_t n, const float* grad_scores, void* stream) {
  if (n == 0) return KGE_OK;
  if (n < 0 || !ent || !rel || !ent_proj || !rel_proj || !grad_ent || !grad_rel || !grad_ent_proj ||
      !grad_rel_proj || !h || !t || !r || !grad_scores)
    return fail(KGE_ERR_ARG, "kge_transd_score_triples_bwd: bad argument");
  if (int e = transd_widths(ent_dim, rel_dim, "kge_transd_score_triples_bwd")) return e;
  DeviceScope device_scope(ent);
  KGE_CUDA_TRY(kge::launch_transd_score_bwd(ent, rel, ent_proj, rel_proj, grad_ent, grad_rel, grad_ent_proj,
                                            grad_rel_proj, ent_dim, rel_dim, h, t, r, n, grad_scores,
                                            static_cast<cudaStream_t>(stream)),
               "transd_score_triples_bwd");
  return KGE_OK;
}

int kge_corrupt_batch(const int64_t* h, const int64_t* t, const int64_t* r, int64_t b,
                      int32_t n_neg, const float* bern_probs, int64_t n_ent, uint64_t seed,
                      uint64_t offset, int64_t* nh, int64_t* nt, void* stream) {
  if (b == 0) return KGE_OK;
  if (b < 0 || n_neg < 1 || n_ent < 1 || !h || !t || !r || !bern_probs || !nh || !nt)
    return fail(KGE_ERR_ARG, "kge_corrupt_batch: bad argument");
  DeviceScope device_scope(h);
  KGE_CUDA_TRY(kge::launch_corrupt_batch(h, t, r, b, n_neg, bern_probs, n_ent, seed, offset, nh, nt,
                                         static_cast<cudaStream_t>(stream)),
               "corrupt_batch");
  return KGE_OK;
}

int kge_margin_loss_fwd(const float* pos, const float* neg, int64_t n, float margin, float* loss,
                        void* stream) {
  if (n == 0) return KGE_OK;
  if (n < 0 || !pos || !neg || !loss) return fail(KGE_ERR_ARG, "kge_margin_loss_fwd: bad argument");
  DeviceScope device_scope(pos);
  KGE_CUDA_TRY(kge::launch_pair_loss_fwd(KGE_LOSS_MARGIN, margin, pos, neg, n, loss,
                                         static_cast<cudaStream_t>(stream)),
               "margin_loss_fwd");
  return KGE_OK;
}

int kge_margin_loss_bwd(const float* pos, const float* neg, int64_t n, float margin,
                        const float* grad_loss, float* grad_pos, float* grad_neg, void* stream) {
  if (n == 0) return KGE_OK;
  if (n < 0 || !pos || !neg || !grad_loss || !grad_pos || !grad_neg)
    return fail(KGE_ERR_ARG, "kge_margin_loss_bwd: bad argument");
  DeviceScope device_scope(pos);
  KGE_CUDA_TRY(kge::launch_pair_loss_bwd(KGE_LOSS_MARGIN, margin, pos, neg, n, grad_loss, grad_pos, grad_neg,
                                         static_cast<cudaStream_t>(stream)),
               "margin_loss_bwd");
  return KGE_OK;
}

int kge_pair_loss_fwd(int kind, const float* pos, const float* neg, int64_t n, float* loss, void* stream) {
  if (kind != KGE_LOSS_LOGISTIC && kind != KGE_LOSS_BCE) return fail(KGE_ERR_ARG, "kge_pair_loss_fwd: unknown loss kind");
  if (n == 0) return KGE_OK;
  if (n < 0 || !pos || !neg || !loss) return fail(KGE_ERR_ARG, "kge_pair_loss_fwd: bad argument");
  DeviceScope device_scope(pos);
  KGE_CUDA_TRY(kge::launch_pair_loss_fwd(kind, 0.f, pos, neg, n, loss, static_cast<cudaStream_t>(stream)),
               "pair_loss_fwd");
  return KGE_OK;
}

int kge_pair_loss_bwd(int kind, const float* pos, const float* neg, int64_t n, const float* grad_loss,
                      float* grad_pos, float* grad_neg, void* stream) {
  if (kind != KGE_LOSS_LOGISTIC && kind != KGE_LOSS_BCE) return fail(KGE_ERR_ARG, "kge_pair_loss_bwd: unknown loss kind");
  if (n == 0) return KGE_OK;
  if (n < 0 || !pos || !neg || !grad_loss || !grad_pos || !grad_neg)
    return fail(KGE_ERR_ARG, "kge_pair_loss_bwd: bad argument");
  DeviceScope device_scope(pos);
  KGE_CUDA_TRY(kge::launch_pair_loss_bwd(kind, 0.f, pos, neg, n, grad_loss, grad_pos, grad_neg,
                                         static_cast<cudaStream_t>(stream)),
               "pair_loss_bwd");
  return KGE_OK;
}

int kge_margin_step_fwd(const kge_margin_step_args_t* a) {
  if (!step_ok(a)) return fail(KGE_ERR_ARG, "kge_margin_step_fwd: bad argument");
  DeviceScope device_scope(a->tb.ent0);
  KGE_CUDA_TRY(kge::launch_margin_step_fwd(to_step(a), static_cast<cudaStream_t>(a->stream)),
               "margin_step_fwd");
  return KGE_OK;
}

int kge_margin_step_bwd(const kge_margin_step_args_t* a, const kge_grads_t* g,
                        const float* grad_loss) {
  if (!step_ok(a) || !step_grads_ok(a, g) || !grad_loss || !shard_grads_ok(a))
    return fail(KGE_ERR_ARG, "kge_margin_step_bwd: bad argument");
  DeviceScope device_scope(a->tb.ent0);
  KGE_CUDA_TRY(kge::launch_margin_step_bwd(to_step(a), to_grads(g), grad_loss,
                                           static_cast<cudaStream_t>(a->stream)),
               "margin_step_bwd");
  return KGE_OK;
}

int kge_corrupt_batch_rel(const int64_t* h, const int64_t* t, const int64_t* r, int64_t b, int32_t n_neg,
                          const float* bern_probs, int64_t n_ent, int64_t n_rel, float rel_share, uint64_t seed,
                          uint64_t offset, int64_t* nh, int64_t* nt, int64_t* nr, void* stream) {
  if (b < 0 || n_neg < 1 || n_ent < 1 || !rel_draw_ok(n_rel, rel_share))
    return fail(KGE_ERR_ARG, "kge_corrupt_batch_rel: bad argument");
  if (b == 0) return KGE_OK;
  if (!h || !t || !r || !bern_probs || !nh || !nt || !nr)
    return fail(KGE_ERR_ARG, "kge_corrupt_batch_rel: null pointer");
  DeviceScope device_scope(h);
  KGE_CUDA_TRY(kge::launch_corrupt_batch_rel(h, t, r, b, n_neg, bern_probs, n_ent, n_rel, rel_share, seed, offset,
                                             nh, nt, nr, static_cast<cudaStream_t>(stream)),
               "corrupt_batch_rel");
  return KGE_OK;
}

int kge_rel_step_fwd(const kge_rel_step_args_t* a) {
  if (!rel_step_ok(a)) return fail(KGE_ERR_ARG, "kge_rel_step_fwd: bad argument");
  DeviceScope device_scope(a->base.tb.ent0);
  KGE_CUDA_TRY(kge::launch_margin_step_fwd(to_rel_step(a), static_cast<cudaStream_t>(a->base.stream)),
               "rel_step_fwd");
  return KGE_OK;
}

int kge_rel_step_bwd(const kge_rel_step_args_t* a, const kge_grads_t* g, const float* grad_loss) {
  if (!rel_step_ok(a) || !step_grads_ok(&a->base, g) || !grad_loss || !shard_grads_ok(&a->base))
    return fail(KGE_ERR_ARG, "kge_rel_step_bwd: bad argument");
  DeviceScope device_scope(a->base.tb.ent0);
  KGE_CUDA_TRY(kge::launch_margin_step_bwd(to_rel_step(a), to_grads(g), grad_loss,
                                           static_cast<cudaStream_t>(a->base.stream)),
               "rel_step_bwd");
  return KGE_OK;
}

int kge_pos_step_fwd(const kge_pos_step_args_t* a) {
  if (!a) return fail(KGE_ERR_ARG, "kge_pos_step_fwd: bad argument");
  DeviceScope device_scope(a->base.tb.ent0);   // before pos_step_ok, which may read offsets
  if (!pos_step_ok(a)) return fail(KGE_ERR_ARG, "kge_pos_step_fwd: bad argument");
  KGE_CUDA_TRY(kge::launch_margin_step_fwd(to_step(&a->base), static_cast<cudaStream_t>(a->base.stream),
                                           to_pos_csr(a)),
               "pos_step_fwd");
  return KGE_OK;
}

int kge_pos_step_bwd(const kge_pos_step_args_t* a, const kge_grads_t* g, const float* grad_loss) {
  if (!a || !step_grads_ok(&a->base, g) || !grad_loss || !shard_grads_ok(&a->base))
    return fail(KGE_ERR_ARG, "kge_pos_step_bwd: bad argument");
  DeviceScope device_scope(a->base.tb.ent0);   // before pos_step_ok, which may read offsets
  if (!pos_step_ok(a)) return fail(KGE_ERR_ARG, "kge_pos_step_bwd: bad argument");
  KGE_CUDA_TRY(kge::launch_margin_step_bwd(to_step(&a->base), to_grads(g), grad_loss,
                                           static_cast<cudaStream_t>(a->base.stream), to_pos_csr(a)),
               "pos_step_bwd");
  return KGE_OK;
}

int kge_scatter_rows_add(int model, float* grad0, float* grad1, int64_t ent_lo, int64_t n_rows, int dim,
                         const int64_t* idx, int64_t n, const float* rows, void* stream) {
  const int planes = kge_cand_planes(model);
  if (planes == 0) return fail(KGE_ERR_ARG, "kge_scatter_rows_add: unknown model");
  if (n < 0 || n_rows < 0 || dim < 1) return fail(KGE_ERR_ARG, "kge_scatter_rows_add: bad sizes");
  if (n == 0 || n_rows == 0) return KGE_OK;
  if (!grad0 || !idx || !rows || (planes >= 2 && !grad1))
    return fail(KGE_ERR_ARG, "kge_scatter_rows_add: null pointer");
  DeviceScope device_scope(grad0);
  KGE_CUDA_TRY(kge::launch_scatter_rows_add(grad0, grad1, planes, ent_lo, n_rows, dim, idx, n, rows,
                                            static_cast<cudaStream_t>(stream)),
               "scatter_rows_add");
  return KGE_OK;
}

int kge_scan_timing_enable(int on) {
  std::lock_guard<std::mutex> lock(g_timing_mu);
  g_timing_on = on != 0;
  return KGE_OK;
}

int kge_scan_timing_read(int kind, int64_t* launches, double* total_ms) {
  if (kind < 0 || kind >= TIMING_KINDS) return fail(KGE_ERR_ARG, "kge_scan_timing_read: bad kind");
  std::vector<std::pair<cudaEvent_t, cudaEvent_t>> ev;
  {
    std::lock_guard<std::mutex> lock(g_timing_mu);
    ev.swap(g_timing_events[kind]);
  }
  double total = 0.0;
  int rc = KGE_OK;
  for (auto& pr : ev) {
    cudaError_t e = cudaEventSynchronize(pr.second);
    float ms = 0.f;
    if (e == cudaSuccess) e = cudaEventElapsedTime(&ms, pr.first, pr.second);
    if (e != cudaSuccess) rc = fail_cuda(e, "scan timing");
    total += ms;
    cudaEventDestroy(pr.first);
    cudaEventDestroy(pr.second);
  }
  if (launches) *launches = (int64_t)ev.size();
  if (total_ms) *total_ms = total;
  return rc;
}

}  // extern "C"
