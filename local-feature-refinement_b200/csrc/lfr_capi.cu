// lfr_capi.cu — the C ABI of include/lfr.h for the CUDA backend: plan
// construction (problem -> HBM, size-bucketed launch schedule), the solve
// launches, and result download.  No CPU fallback: every entry point that
// computes fails with LFR_ENODEV / LFR_ECUDA when no device is usable.
#include <algorithm>
#include <cassert>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <unordered_set>
#include <vector>

#include "../../include/lfr_graph.h"
#include "lfr_cut.h"
#include "lfr_cut.cuh"
#include "lfr_diff.cuh"
#include "lfr_graph.cuh"
#include "lfr_record.cuh"
#include "lfr_solution.cuh"
#include "lfr_solve_cta.cuh"
#include "lfr_solve_warp.cuh"
#include "lfr_solve_warp2.cuh"
#include "lfr_start.cuh"
#include "lfr_join.h"
#include "lfr_wire.cuh"

namespace {

thread_local std::string g_last_error;

// host-side timeline of the calling thread's last lfr_solve(): microseconds since the call began at
// {small uploads queued, schedule built, plan filled, kernels queued, stats back, return}
thread_local double g_host_marks[8] = {};
thread_local std::chrono::steady_clock::time_point g_host_t0;
inline void host_mark(int i) {
  g_host_marks[i] = std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now() - g_host_t0).count();
}

int fail(int code, const std::string& msg) {
  g_last_error = msg;
  return code;
}

int cuda_code(cudaError_t e) {
  if (e == cudaErrorNoDevice || e == cudaErrorInsufficientDriver || e == cudaErrorInvalidDevice) return LFR_ENODEV;
  if (e == cudaErrorMemoryAllocation) return LFR_ENOMEM;
  return LFR_ECUDA;
}

#define LFR_CUDA(call)                                                              \
  do {                                                                              \
    cudaError_t err__ = (call);                                                     \
    if (err__ != cudaSuccess)                                                       \
      return fail(cuda_code(err__), std::string(#call) + ": " + cudaGetErrorString(err__)); \
  } while (0)

#define LFR_TRY(expr)        \
  do {                       \
    const int rc__ = (expr); \
    if (rc__) return rc__;   \
  } while (0)

constexpr int kMaxSmemPerBlock = 227 * 1024;
// Components with more unknowns than this (and <= 32) take the two-warp tile kernel <64, 32> instead of
// the one-warp register kernel; 32 = never.  Overridden per plan by LFR_TILE_FROM_N.
constexpr int kTileFromDefault = 32;
// warps per SM of the warp-register tier's queue kernel (LFR_DBG_WARP2_WARPS_SHIFT overrides, up to
// lfr::kWarp2QueueMaxWarps)
constexpr int kWarp2QueueWarpsDefault = 8;
constexpr int kScheduleThreadsMax = 8;  // host threads that classify the dispatch list (build_schedule)
constexpr int kMaxStreams = 12;

lfr::DevConsts make_consts(const lfr_options& o) {
  lfr::DevConsts K;
  K.bound = o.bound;
  K.cauchy_b = o.cauchy_a * o.cauchy_a;
  K.cauchy_c = 1.0 / K.cauchy_b;
  K.tukey_a2 = o.tukey_a * o.tukey_a;
  K.tukey_inv_a2 = 1.0 / K.tukey_a2;
  if (o.tukey_variant == 2) {
    K.tukey_rho0 = K.tukey_a2 / 3.0;
    K.tukey_rho1 = 1.0;
  } else {
    K.tukey_rho0 = K.tukey_a2 / 6.0;
    K.tukey_rho1 = 0.5;
  }
  K.f_tol = o.function_tolerance;
  K.g_tol = o.gradient_tolerance;
  K.p_tol = o.parameter_tolerance;
  K.radius0 = o.initial_trust_region_radius;
  K.radius_max = o.max_trust_region_radius;
  K.radius_min = o.min_trust_region_radius;
  K.min_rel_decrease = o.min_relative_decrease;
  K.min_diag = o.min_lm_diagonal;
  K.max_diag = o.max_lm_diagonal;
  K.ls_suff = o.line_search_sufficient_function_decrease;
  K.ls_max_contraction = o.max_line_search_step_contraction;
  K.ls_min_contraction = o.min_line_search_step_contraction;
  K.ls_min_step = o.min_line_search_step_size;
  K.max_iter = o.max_num_iterations;
  K.max_invalid = o.max_num_consecutive_invalid_steps;
  K.max_ls_iter = o.max_num_line_search_step_size_iterations;
  K.linear_solver = o.linear_solver;
  return K;
}

// Grow-only device buffer: lfr_solve() re-uses its workspace across calls, so a
// steady stream of solves performs no cudaMalloc/cudaFree.
struct DevBuf {
  void* p = nullptr;
  size_t cap = 0;
  int reserve(size_t bytes) {
    if (bytes <= cap) return LFR_OK;
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
    const size_t want = bytes + bytes / 8 + 256;
    cudaError_t e = cudaMalloc(&p, want);
    if (e != cudaSuccess) return fail(cuda_code(e), std::string("cudaMalloc: ") + cudaGetErrorString(e));
    cap = want;
    return LFR_OK;
  }
  void release() {
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
  }
  template <typename T>
  T* as() const { return static_cast<T*>(p); }
};

// The solve kernels.  The schedule builder picks one per launch; launch_solve has one launch statement each.
enum class Kernel : uint8_t {
  kWarp2x4_8, kWarp2x4_16, kWarp2x1_32,                // solve_warp2_kernel<WARPS, NREG>
  kQueue,                                              // solve_warp2_queue_kernel
  kTile64x32, kTile64x48, kTile64x64, kTile128x80,     // solve_tile_kernel<T, NREG>
  kWarp4, kWarp1,                                      // solve_warp_kernel<WARPS> (shared-memory Cholesky)
  kCta2, kCta3, kCta4,                                 // solve_cta_kernel<256, MINB>
  kCount
};
inline bool is_cta(Kernel k) { return k >= Kernel::kCta2; }

// Where a kernel reads its edge records: staged into shared memory from DevProblem::edges (the HBM copy
// or the caller's pinned array), from the HBM copy by global index, or from the CTA tier's own arrays
// that cta_prepare_kernel fills.
enum class Edges : uint8_t { kStaged, kGlobal, kPrepared };

struct KernelInfo {
  const void* fn;  // for cudaFuncSetAttribute
  int threads;     // per component; a CTA runs Launch::warps components
  int per_cta;     // components per CTA (the queue: set per launch)
  Edges edges;
  int smem_max;    // dynamic shared memory to allow
  int label;       // what LFR_SCHED_DUMP prints: a bucket's variant code, or a CTA kernel's MINB
};

const KernelInfo kKernels[] = {
    {(const void*)lfr::solve_warp2_kernel<4, 8>, 32, 4, Edges::kStaged, kMaxSmemPerBlock, 8},
    {(const void*)lfr::solve_warp2_kernel<4, 16>, 32, 4, Edges::kStaged, kMaxSmemPerBlock, 16},
    {(const void*)lfr::solve_warp2_kernel<1, 32>, 32, 1, Edges::kStaged, kMaxSmemPerBlock, 32},
    {(const void*)lfr::solve_warp2_queue_kernel, 32, 0, Edges::kStaged, kMaxSmemPerBlock, 0},
    {(const void*)lfr::solve_tile_kernel<64, 32>, 64, 1, Edges::kStaged, kMaxSmemPerBlock, 132},
    {(const void*)lfr::solve_tile_kernel<64, 48>, 64, 1, Edges::kStaged, kMaxSmemPerBlock, 48},
    {(const void*)lfr::solve_tile_kernel<64, 64>, 64, 1, Edges::kStaged, kMaxSmemPerBlock, 64},
    {(const void*)lfr::solve_tile_kernel<128, 80>, 128, 1, Edges::kStaged, kMaxSmemPerBlock, 80},
    {(const void*)lfr::solve_warp_kernel<4>, 32, 4, Edges::kGlobal, kMaxSmemPerBlock, 0},
    {(const void*)lfr::solve_warp_kernel<1>, 32, 1, Edges::kGlobal, kMaxSmemPerBlock, 0},
    {(const void*)lfr::solve_cta_kernel<256, 2>, 256, 1, Edges::kPrepared, 200 * 1024, 2},
    {(const void*)lfr::solve_cta_kernel<256, 3>, 256, 1, Edges::kPrepared, 200 * 1024, 3},
    {(const void*)lfr::solve_cta_kernel<256, 4>, 256, 1, Edges::kPrepared, 200 * 1024, 4},
};
static_assert(sizeof(kKernels) / sizeof(kKernels[0]) == (size_t)Kernel::kCount, "one entry per kernel");
inline const KernelInfo& info(Kernel k) { return kKernels[(int)k]; }

// One kernel launch of a solve: `n` members from `offset`, `warps` of them per CTA, each in `bytes` of
// dynamic shared memory.
//  - per-bucket kernels: dispatch slots in the list buffer; `bytes` is the layout of the members' maxima
//    (emax, ncmax, n2max);
//  - the queue: entries of two words in the list buffer, `warps` per SM, slots of `bytes`;
//  - the CTA tier: components of L_comps, one per CTA; `bytes` holds the CG vectors of the largest
//    (`max_free` free nodes, the first `smem_vecs` of p, w, r, z, y and the preconditioner).
struct Launch {
  Kernel kernel = Kernel::kCount;
  uint32_t offset = 0, n = 0;
  int emax = 0, ncmax = 0, n2max = 0, bytes = 0, warps = 1;
  uint32_t max_free = 0;
  int smem_vecs = 0;
};

int validate(const lfr_problem* p) {
  if (!p) return fail(LFR_EINVAL, "problem is NULL");
  if (p->n_nodes && (!p->row_ptr || !p->track || !p->comp || !p->is_root))
    return fail(LFR_EINVAL, "NULL per-node array");
  if (p->n_components && (!p->comp_ptr || !p->comp_nodes)) return fail(LFR_EINVAL, "NULL component list");
  if (p->n_nodes && p->row_ptr[p->n_nodes] != p->n_edges) return fail(LFR_EINVAL, "row_ptr[n_nodes] != n_edges");
  if (p->n_edges && !p->edges) return fail(LFR_EINVAL, "edges is NULL");
  if (p->n_edges >= (1ull << 32)) return fail(LFR_EUNSUPPORTED, "more than 2^32 directed edges");
  // the per-edge checks (dst range, self edges, a component node list that disagrees with `comp`)
  // run on the device as every tier classifies its edges (classify_edge), so the host never walks the
  // 80-byte records.
  return LFR_OK;
}

}  // namespace

struct lfr_plan {
  int device = 0;
  lfr_options opt;
  lfr::DevConsts K;
  uint32_t N = 0, C = 0;
  uint64_t E = 0;
  uint32_t total_slots = 0;
  DevBuf row_ptr, edges, track, comp, is_root, comp_ptr, comp_nodes, local_of, pos, pos_init, stats, cycles, times, lists;
  // `stats` is one block (one memset, one D2H copy): cost0[Cp] cost1[Cp] iter[Cp] term[Cp] ls[Cp] kept[Cp] err[2] pull[2 x u64]
  uint32_t Cp = 0;               // C rounded up to an even count
  bool pos_is_staged = false;    // lfr_solve(): the start point was uploaded straight into `pos`
  void* h_stage = nullptr;       // pinned host staging for the stats block
  size_t h_stage_cap = 0;
  double* d_cost0() const { return stats.as<double>(); }
  double* d_cost1() const { return stats.as<double>() + Cp; }
  int32_t* d_iter() const { return reinterpret_cast<int32_t*>(stats.as<double>() + 2 * (size_t)Cp); }
  int32_t* d_term() const { return d_iter() + Cp; }
  uint32_t* d_ls() const { return reinterpret_cast<uint32_t*>(d_term() + Cp); }
  uint32_t* d_kept() const { return d_ls() + Cp; }
  int* d_err() const { return reinterpret_cast<int*>(d_kept() + Cp); }
  unsigned long long* d_pull() const { return reinterpret_cast<unsigned long long*>(d_err() + 2); }  // {ticketed, arrived} bytes
  size_t stats_bytes() const { return 16 * (size_t)Cp + 16 * (size_t)Cp + 8 + 16; }
  std::vector<Launch> launches;       // in launch order: the CTA tier, the queue, the buckets
  std::vector<uint32_t> w2_slots;     // build_schedule scratch: the queue's members
  DevBuf queue_ctr;                   // two words per queue launch (solve_warp2_queue_kernel)
  int n_sms = 0;
  int num_launches() const { return (int)launches.size(); }
  std::vector<uint32_t> comp_size;  // nodes per dispatch slot
  std::vector<uint32_t> list_host;
  // CTA tier (block-Jacobi PCG): components with more than kMaxWarpN2 unknowns, or all with linear_solver = 2
  struct SchedDim { int e, nc, n2; };
  std::vector<uint16_t> sched_key;        // build_schedule scratch: (route, shared-memory class) of every slot
  std::vector<SchedDim> sched_dim;
  // the CTA tier's components by size class, in dispatch order inside a class
  std::vector<uint32_t> large_slots;
  std::vector<uint64_t> large_cand;       // candidate out-edges of each large component (row_ptr sums)
  std::vector<uint32_t> large_free;       // its non-root nodes (upper bound of the free nodes)
  std::vector<uint64_t> large_ell;        // its sliced-ELL slots (32 x the largest candidate out-degree of every 32-node slice)
  std::vector<lfr::CtaComp> L_comps_host;
  uint32_t n_large = 0;
  DevBuf L_comps, L_rec, L_meta, L_inlist, L_twin, L_fdst, L_bE01, L_bE23, L_fdstE, L_ell_base, L_scr, L_q, L_node, L_outptr, L_inptr, L_freeof, L_x, L_xc, L_lof, L_vec;
  uint64_t L_total_free = 0;
  uint32_t n_solved = 0;
  bool profile = false;
  // lfr_solve() zero-copy: staging tiers read the caller's pinned edge array / write the caller's
  // pinned positions directly (device-side addresses of those host buffers), nullptr = through HBM
  const float4* zc_edges = nullptr;
  double* zc_positions = nullptr;
  const uint8_t* slot_owner = nullptr;  // lfr_solve_multi(): owner[c] of every dispatch slot, this plan solves owner == owner_id
  uint8_t owner_id = 0;
  bool edges_in_hbm = false;       // the edge array was (or is being) copied to `edges`
  cudaStream_t copy_stream = nullptr;
  cudaEvent_t ev_edges = nullptr;  // bulk edge copy done (only the non-staging tiers wait for it)
  cudaEvent_t ev_small = nullptr;  // fork / join of the second upload stream
  cudaEvent_t ev_prep = nullptr;   // small arrays + local_of ready (CTA-tier preparation on the copy stream)
  bool cta_from_hbm = false;       // zero-copy solve whose CTA tier reads the bulk HBM copy of the edge array
  cudaStream_t streams[kMaxStreams] = {};
  cudaEvent_t ev_fork = nullptr, ev_join[kMaxStreams] = {};
  int n_streams = 0;
  // a plan built from matches (lfr_plan_create_from_matches): the host copies of the stage's arrays
  struct GraphArrays {
    std::vector<uint32_t> row_ptr, track, comp, comp_ptr, comp_nodes, comp_order, node_image, node_feat;
    std::vector<uint8_t> is_root;
  };
  std::unique_ptr<GraphArrays> graph;
  // ... and on the device, for lfr_plan_encode_solution(): the node ids (8 B per node), the image count of
  // the input, the encoder's scratch and its output (grow-only: repeated encodes allocate nothing)
  DevBuf node_image, node_feat, enc_scratch, enc_cub, enc_out;
  uint32_t n_images = 0;
  // lfr_plan_fix_images() / lfr_plan_keep_solution(): the constant mask the tiers read in place of
  // `is_root` (reference roots OR nodes of fixed images OR kept nodes) and its host copy for the schedule
  // builder; never allocated for a plan without one.  Its two inputs are kept apart, so that each call
  // replaces only its own: the per-image mask (empty until lfr_plan_fix_images()) and the per-node kept
  // flags (allocated by the first lfr_plan_keep_solution() or lfr_plan_update_solution(), whose held flags
  // they are then: the last of the two calls wins)
  DevBuf const_mask;
  std::vector<uint8_t> const_host;
  std::vector<uint8_t> fixed_host;
  DevBuf kept;

  lfr::CtaArrays cta_arrays() const {
    lfr::CtaArrays A;
    A.rec = L_rec.as<float4>();
    A.meta = L_meta.as<uint32_t>();
    A.inlist = L_inlist.as<uint32_t>();
    A.twin = L_twin.as<uint32_t>();
    A.fdst = L_fdst.as<int32_t>();
    A.bE01 = L_bE01.as<double2>();
    A.bE23 = L_bE23.as<double2>();
    A.fdstE = L_fdstE.as<int32_t>();
    A.ell_base = L_ell_base.as<uint32_t>();
    A.scr = L_scr.as<double>();
    A.q = L_q.as<double>();
    A.node = L_node.as<uint32_t>();
    A.outptr = L_outptr.as<uint32_t>();
    A.inptr = L_inptr.as<uint32_t>();
    A.freeof = L_freeof.as<int32_t>();
    A.x = L_x.as<double>();
    A.xc = L_xc.as<double>();
    A.lof = L_lof.as<uint32_t>();
    A.vec = L_vec.as<double>();
    A.total_free = L_total_free;
    return A;
  }

  lfr::DevProblem dev() const {
    lfr::DevProblem P;
    P.n_nodes = N;
    P.row_ptr = row_ptr.as<uint32_t>();
    P.edges = edges.as<float4>();
    P.track = track.as<uint32_t>();
    P.comp = comp.as<uint32_t>();
    P.is_root = const_mask.p ? const_mask.as<uint8_t>() : is_root.as<uint8_t>();
    P.comp_ptr = comp_ptr.as<uint32_t>();
    P.comp_nodes = comp_nodes.as<uint32_t>();
    P.local_of = local_of.as<uint32_t>();
    P.positions = pos.as<double>();
    P.positions_out = zc_positions ? zc_positions : pos.as<double>();
    P.pull_ctr = d_pull();
    P.pull_window = 0;  // set by launch_solve for zero-copy staging only
    P.st_iter = d_iter();
    P.st_term = d_term();
    P.st_cost0 = d_cost0();
    P.st_cost1 = d_cost1();
    P.st_ls = d_ls();
    P.st_kept = d_kept();
    P.st_cycles = profile ? cycles.as<unsigned long long>() : nullptr;
    P.st_times = profile ? times.as<unsigned long long>() : nullptr;
    P.err_flag = d_err();
    return P;
  }
};

namespace {

void free_plan(lfr_plan* pl) {
  if (!pl) return;
  DevBuf* bufs[] = {&pl->row_ptr, &pl->edges, &pl->track, &pl->comp, &pl->is_root, &pl->comp_ptr, &pl->comp_nodes,
                    &pl->local_of, &pl->pos, &pl->pos_init, &pl->stats, &pl->cycles, &pl->times, &pl->lists, &pl->L_comps, &pl->L_rec, &pl->L_meta,
                    &pl->L_inlist, &pl->L_twin, &pl->L_fdst, &pl->L_bE01, &pl->L_bE23, &pl->L_fdstE, &pl->L_ell_base, &pl->L_scr, &pl->L_q, &pl->L_node, &pl->L_outptr, &pl->L_inptr, &pl->L_freeof,
                    &pl->L_x, &pl->L_xc, &pl->L_lof, &pl->L_vec, &pl->node_image, &pl->node_feat, &pl->enc_scratch,
                    &pl->enc_cub, &pl->enc_out, &pl->queue_ctr, &pl->const_mask, &pl->kept};
  for (DevBuf* b : bufs) b->release();
  if (pl->h_stage) cudaFreeHost(pl->h_stage);
  for (int i = 0; i < pl->n_streams; ++i) {
    if (pl->streams[i]) cudaStreamDestroy(pl->streams[i]);
    if (pl->ev_join[i]) cudaEventDestroy(pl->ev_join[i]);
  }
  if (pl->ev_fork) cudaEventDestroy(pl->ev_fork);
  if (pl->ev_edges) cudaEventDestroy(pl->ev_edges);
  if (pl->ev_small) cudaEventDestroy(pl->ev_small);
  if (pl->ev_prep) cudaEventDestroy(pl->ev_prep);
  if (pl->copy_stream) cudaStreamDestroy(pl->copy_stream);
  delete pl;
}

template <typename T>
int upload(DevBuf* d, const T* h, size_t count, cudaStream_t s) {
  LFR_TRY(d->reserve(std::max<size_t>(count, 1) * sizeof(T)));
  if (count) LFR_CUDA(cudaMemcpyAsync(d->p, h, count * sizeof(T), cudaMemcpyHostToDevice, s));
  return LFR_OK;
}

// The solve's launch list (pl->launches).  Components are grouped by the shared memory one warp needs
// for them, so small tracks run at high occupancy and the few large components do not dictate the
// carve-up of everyone else.  The CTA tier launches first, one launch per size class; then the register
// warp tier's four-warp members in persistent queue launches (where one of them has more than 16
// unknowns), then one launch per (route, shared-memory class) bucket, largest components first.
int build_schedule(lfr_plan* pl, const lfr_problem* p) {
  // shared-memory classes of a launch (finer classes — one per "one more CTA fits an SM" boundary — mean
  // more launches for the same resident work)
  static const int kClass[] = {2048, 3072, 4096, 6144, 8192, 12288, 16384, 24576, 32768, 57344, kMaxSmemPerBlock};
  constexpr int n_class = sizeof(kClass) / sizeof(kClass[0]);
  // the route of a component off the CTA tier: a register class (NREG 8..32), a tile kernel, or the
  // shared-memory Cholesky warp kernel; inside a shared-memory class the last route launches first
  enum Route { kReg8, kReg16, kReg24, kReg32, kTile32, kTile48, kTile64, kTile80, kCholesky, kRoutes };
  // a route's kernel where four of its slots fit a CTA, and where they do not (the register classes
  // above 16 unknowns have no four-warp kernel of their own: the queue runs them)
  static const Kernel kFour[kRoutes] = {Kernel::kWarp2x4_8, Kernel::kWarp2x4_16, Kernel::kQueue, Kernel::kQueue,
                                        Kernel::kTile64x32, Kernel::kTile64x48, Kernel::kTile64x64, Kernel::kTile128x80,
                                        Kernel::kWarp4};
  static const Kernel kOne[kRoutes] = {Kernel::kWarp2x1_32, Kernel::kWarp2x1_32, Kernel::kWarp2x1_32, Kernel::kWarp2x1_32,
                                       Kernel::kTile64x32, Kernel::kTile64x48, Kernel::kTile64x64, Kernel::kTile128x80,
                                       Kernel::kWarp1};
  constexpr int kKeys = kRoutes * n_class;
  constexpr uint16_t kNoKey = 0xffff;
  auto is_tile = [](int r) { return r >= kTile32 && r <= kTile80; };
  auto fits_four = [](int bytes) { return 4 * bytes <= kMaxSmemPerBlock; };
  const int dbg = pl->opt.debug_flags;
  const bool no_tile = (dbg & LFR_DBG_NO_TILE) != 0;
  // components with more than tile_from unknowns (and <= 32) go to the two-warp tile kernel
  // instead of the one-warp kernel (their edge evaluation is split over 64 threads)
  const int tf = (dbg >> LFR_DBG_TILE_FROM_SHIFT) & 0xff;
  const int tile_from = no_tile ? 32 : (tf ? tf : kTileFromDefault);
  const bool force_v1 = (dbg & LFR_DBG_FORCE_SMEM_CHOLESKY) != 0;
  const bool force_pcg = pl->opt.linear_solver == 2;
  auto layout_bytes = [&](int r, int e, int nc, int n2) {
    return (r == kCholesky) ? lfr::WarpLayout(e, nc, n2).total
                            : lfr::RegLayout(e, nc, n2, is_tile(r) ? 64 : 32).total;  // (one layout for both tile widths)
  };
  // This runs on the calling thread while the GPU waits for its first launch: one pass over the
  // components into flat, reused arrays (no per-call allocation once the plan is warm), then a
  // counting sort of the slots by (route, shared-memory class).
  const uint32_t C = p->n_components;
  pl->comp_size.resize(C);
  pl->sched_key.resize(C);
  pl->sched_dim.resize(C);
  pl->n_solved = 0;
  pl->launches.clear();
  pl->large_slots.clear();
  pl->large_cand.clear();
  pl->large_free.clear();
  pl->large_ell.clear();
  const uint32_t* comp_ptr = p->comp_ptr;
  const uint32_t* comp_nodes = p->comp_nodes;
  const uint32_t* row_ptr = p->row_ptr;
  const uint8_t* is_root = p->is_root;
  const uint8_t* owner = pl->slot_owner;
  const uint32_t n_nodes = p->n_nodes;
  uint16_t* key_of = pl->sched_key.data();
  lfr_plan::SchedDim* dim = pl->sched_dim.data();
  // Pass 1 — classify the slots [c0, c1): a pure function of the problem arrays that writes only the
  // per-slot entries of its own range and its own accumulator, so ranges run on separate threads
  // (merged in range order: the schedule does not depend on the thread count).
  struct Acc {
    lfr_plan::SchedDim caps[kKeys] = {};  // maxima of the members
    uint32_t count[kKeys] = {};
    uint32_t fit4[kKeys] = {};            // members whose own slot fits four to a CTA
    uint32_t n_solved = 0;
    std::vector<uint32_t> large_slots, large_free;
    std::vector<uint64_t> large_cand, large_ell;
    int rc = LFR_OK;
    const char* msg = nullptr;
  };
  auto classify = [&](uint32_t c0, uint32_t c1, Acc& A) {
    auto bail = [&](int code, const char* m) {
      A.rc = code;
      A.msg = m;
    };
    for (uint32_t c = c0; c < c1; ++c) {
      const uint32_t beg = comp_ptr[c], end = comp_ptr[c + 1];
      if (end < beg || end > pl->total_slots) return bail(LFR_EINVAL, "comp_ptr not monotone");
      const uint32_t nc = end - beg;
      pl->comp_size[c] = nc;
      key_of[c] = kNoKey;
      if (nc <= 1) continue;  // solve.cc:619-622
      if (owner && owner[c] != pl->owner_id) continue;  // another device's component
      ++A.n_solved;
      uint64_t eup = 0;
      uint32_t nfree = 0;
      for (uint32_t i = beg; i < end; ++i) {
        const uint32_t v = comp_nodes[i];
        if (v >= n_nodes) return bail(LFR_EINVAL, "comp_nodes out of range");
        const uint32_t r0 = row_ptr[v], r1 = row_ptr[v + 1];
        if (r1 < r0) return bail(LFR_EINVAL, "row_ptr not monotone");
        eup += r1 - r0;
        nfree += is_root[v] ? 0 : 1;
      }
      const int n2 = std::max(2 * (int)nfree, 2);
      auto to_cta_tier = [&]() -> bool {
        if (nc > 16383) {
          bail(LFR_EUNSUPPORTED, "component with more than 16383 nodes");
          return false;
        }
        uint64_t slots = 0;
        for (uint32_t i0 = beg; i0 < end; i0 += 32) {
          uint32_t wmax = 0;
          for (uint32_t i = i0; i < std::min(end, i0 + 32); ++i) wmax = std::max(wmax, row_ptr[comp_nodes[i] + 1] - row_ptr[comp_nodes[i]]);
          slots += 32ull * ((wmax + 3u) & ~3u);  // slice width: a multiple of four slots (cta_block_row)
        }
        if (slots > 0xffffffffull) {
          bail(LFR_EUNSUPPORTED, "component too dense for the CTA tier's block layout");
          return false;
        }
        A.large_slots.push_back(c);
        A.large_cand.push_back(eup);
        A.large_free.push_back(nfree);
        A.large_ell.push_back(slots);
        return true;
      };
      if (force_pcg || n2 > lfr::kMaxWarpN2 || nc > (uint32_t)lfr::kMaxWarpNodes || eup > 65535) {
        if (!to_cta_tier()) return;
        continue;
      }
      const int e = std::max<int>(1, (int)eup);
      int r = (n2 <= 8) ? kReg8 : (n2 <= 16 ? kReg16 : (n2 <= 24 ? kReg24 : (n2 <= 32 ? kReg32 : (n2 <= 48 ? kTile48 : (n2 <= 64 ? kTile64 : (n2 <= 80 ? kTile80 : kCholesky))))));
      if (r <= kReg32 && n2 > tile_from && lfr::RegLayout(e, (int)nc, n2, 64).total <= kMaxSmemPerBlock) r = kTile32;
      if (r >= kTile48 && is_tile(r) && (no_tile || lfr::RegLayout(e, (int)nc, n2, 64).total > kMaxSmemPerBlock)) r = kCholesky;
      if (force_v1) r = kCholesky;
      int need = layout_bytes(r, e, (int)nc, n2);
      if (need > kMaxSmemPerBlock && r != kCholesky) {  // the staged records do not fit: the Cholesky warp kernel reads them from global memory
        r = kCholesky;
        need = layout_bytes(r, e, (int)nc, n2);
      }
      if (need > kMaxSmemPerBlock) {
        // a dense, high-degree component (its per-edge scratch alone exceeds one SM's shared
        // memory): the CTA tier keeps its per-edge data in HBM
        if (!to_cta_tier()) return;
        continue;
      }
      int k = 0;
      while (need > kClass[k]) ++k;  // need <= kClass[n_class - 1] here
      const int key = r * n_class + k;
      key_of[c] = (uint16_t)key;
      dim[c] = lfr_plan::SchedDim{e, (int)nc, n2};
      lfr_plan::SchedDim& cb = A.caps[key];
      ++A.count[key];
      A.fit4[key] += fits_four(need);
      cb.e = std::max(cb.e, e);
      cb.nc = std::max(cb.nc, (int)nc);
      cb.n2 = std::max(cb.n2, n2);
    }
  };
  // ranges of about equal node counts; extra threads only where their start-up pays
  // (cost model: ~3 ns per listed node + ~16 ns per slot on one thread, ~50 us to start a helper)
  const uint64_t work_ns = 3ull * pl->total_slots + 16ull * C;
  // (inside an application the helpers cost more than in the stand-alone timing — the CUDA runtime
  // hooks thread creation — so they start only from about half a millisecond of work)
  int n_thr = work_ns < 500000 ? 1 : (int)std::min<uint64_t>(kScheduleThreadsMax, work_ns / 150000);
  if (const char* e = std::getenv("LFR_SCHEDULE_THREADS")) n_thr = std::max(1, std::min(kScheduleThreadsMax, std::atoi(e)));
  std::vector<uint32_t> cut((size_t)n_thr + 1, C);
  cut[0] = 0;
  for (int t = 1; t < n_thr; ++t) {
    const uint32_t want = (uint32_t)((uint64_t)pl->total_slots * t / n_thr);
    cut[t] = (uint32_t)(std::upper_bound(comp_ptr, comp_ptr + C + 1, want) - comp_ptr);
    cut[t] = std::min(C, std::max(cut[t], cut[t - 1]));
  }
  std::vector<Acc> acc((size_t)n_thr);
  {
    std::vector<std::thread> workers;
    for (int t = 1; t < n_thr; ++t) workers.emplace_back([&, t] { classify(cut[t], cut[t + 1], acc[t]); });
    classify(cut[0], cut[1], acc[0]);
    for (std::thread& w : workers) w.join();
  }
  lfr_plan::SchedDim caps[kKeys] = {};
  uint32_t count[kKeys] = {}, fit4[kKeys] = {};
  for (const Acc& A : acc) {  // range order
    if (A.rc != LFR_OK) return fail(A.rc, A.msg);
    pl->n_solved += A.n_solved;
    for (int k = 0; k < kKeys; ++k) {
      count[k] += A.count[k];
      fit4[k] += A.fit4[k];
      caps[k].e = std::max(caps[k].e, A.caps[k].e);
      caps[k].nc = std::max(caps[k].nc, A.caps[k].nc);
      caps[k].n2 = std::max(caps[k].n2, A.caps[k].n2);
    }
  }
  // The CTA tier: one launch per size class by free nodes (upper bound), in dispatch order (largest
  // first) inside a class.  104 bytes of CG vectors per free node in shared memory -> 1 / 2 / 4 / 8
  // components per SM by shared memory; registers cap it at MINB.
  static const uint32_t kClassMaxFree[4] = {0xffffffffu, 1008, 504, 250};
  int minb[4] = {2, 2, 3, 4};
  if (const char* e = std::getenv("LFR_CTA_MINB")) {  // tuning hook: "2,2,3,4"
    int a[4];
    if (std::sscanf(e, "%d,%d,%d,%d", &a[0], &a[1], &a[2], &a[3]) == 4)
      for (int i = 0; i < 4; ++i) minb[i] = std::min(4, std::max(2, a[i]));
  }
  int smem_vecs[4] = {6, 6, 6, 6};
  if (const char* e = std::getenv("LFR_CTA_SMEM_VECS")) {  // tuning hook: "6,6,6,6"
    int a[4];
    if (std::sscanf(e, "%d,%d,%d,%d", &a[0], &a[1], &a[2], &a[3]) == 4)
      for (int i = 0; i < 4; ++i) smem_vecs[i] = std::min(6, std::max(0, a[i]));
  }
  auto class_of = [&](uint32_t nfree) { return nfree > kClassMaxFree[1] ? 0 : (nfree > kClassMaxFree[2] ? 1 : (nfree > kClassMaxFree[3] ? 2 : 3)); };
  for (int cls = 0; cls < 4; ++cls) {
    Launch g;
    g.kernel = minb[cls] >= 4 ? Kernel::kCta4 : (minb[cls] == 3 ? Kernel::kCta3 : Kernel::kCta2);
    g.offset = (uint32_t)pl->large_slots.size();
    g.smem_vecs = smem_vecs[cls];
    for (const Acc& A : acc)
      for (size_t i = 0; i < A.large_slots.size(); ++i) {
        if (class_of(A.large_free[i]) != cls) continue;
        pl->large_slots.push_back(A.large_slots[i]);
        pl->large_cand.push_back(A.large_cand[i]);
        pl->large_free.push_back(A.large_free[i]);
        pl->large_ell.push_back(A.large_ell[i]);
        g.max_free = std::max(g.max_free, A.large_free[i]);
      }
    g.n = (uint32_t)pl->large_slots.size() - g.offset;
    if (!g.n) continue;
    // the first `smem_vecs` of p, w, r, z, y (2 doubles per free node each) and the preconditioner (3)
    const int per_node = std::min(g.smem_vecs, 5) * 2 + (g.smem_vecs >= 6 ? 3 : 0);
    g.bytes = (int)std::min<uint64_t>(info(g.kernel).smem_max, (uint64_t)g.max_free * per_node * sizeof(double));
    pl->launches.push_back(g);
  }
  // The other routes, per (route, shared-memory class) key: one launch over the union of the members'
  // maxima or, where that overflows, one per member.  The register classes' members of four-warp
  // launches go to the queue instead where one of them has more than 16 unknowns: without one the
  // per-bucket kernels run 12 warps per SM at 168 registers, which the queue kernel (255 registers for
  // all four NREG paths) cannot (DESIGN §4).
  int bytes[kKeys];
  uint32_t four[kKeys];  // members in four-warp launches
  bool wide = false;
  for (int key = 0; key < kKeys; ++key) {
    const int r = key / n_class;
    bytes[key] = count[key] ? layout_bytes(r, caps[key].e, caps[key].nc, caps[key].n2) : 0;
    four[key] = bytes[key] > kMaxSmemPerBlock ? fit4[key] : (fits_four(bytes[key]) ? count[key] : 0);
    wide = wide || ((r == kReg24 || r == kReg32) && four[key]);
  }
  auto queued = [&](int key) { return wide && key / n_class <= kReg32 ? four[key] : 0u; };
  auto slot_of = [&](int key, uint32_t c) {  // a member's slot: its bucket's, or its own where that overflows
    return bytes[key] <= kMaxSmemPerBlock ? bytes[key] : layout_bytes(key / n_class, dim[c].e, dim[c].nc, dim[c].n2);
  };
  // the bucket lists: largest shared-memory class first, within a class the last route first, ascending
  // slot index inside a bucket; the queue's members in ascending slot index
  uint32_t start[kKeys], total = 0;
  for (int k = n_class - 1; k >= 0; --k)
    for (int r = kRoutes - 1; r >= 0; --r) {
      start[r * n_class + k] = total;
      total += count[r * n_class + k] - queued(r * n_class + k);
    }
  pl->list_host.resize(total);
  std::vector<uint32_t>& q = pl->w2_slots;
  q.clear();
  {
    uint32_t fill[kKeys];
    std::memcpy(fill, start, sizeof(fill));
    uint32_t* list = pl->list_host.data();
    for (uint32_t c = 0; c < C; ++c) {
      const int key = key_of[c];
      if (key == kNoKey) continue;
      if (wide && key / n_class <= kReg32 && fits_four(slot_of(key, c)))
        q.push_back(c);
      else
        list[fill[key]++] = c;
    }
  }
  // The queue (solve_warp2_queue_kernel), each entry {slot, own layout sizes}: one launch takes every
  // member whose own layout fits a slot at W warps per SM; the rest (if any) go to a second at as many
  // warps as its largest member allows (>= 4: they fit four to a CTA).
  if (!q.empty()) {
    const int ww = (dbg >> LFR_DBG_WARP2_WARPS_SHIFT) & 0xf;
    const int W = ww ? std::min(ww, lfr::kWarp2QueueMaxWarps) : kWarp2QueueWarpsDefault;
    const int cap = (kMaxSmemPerBlock / W) & ~15;
    for (int pass = 0; pass < 2; ++pass) {
      Launch g;
      g.kernel = Kernel::kQueue;
      g.offset = (uint32_t)pl->list_host.size();
      for (uint32_t c : q) {
        const int b = lfr::RegLayout(dim[c].e, dim[c].nc, dim[c].n2, 32).total;
        if ((b <= cap) != (pass == 0)) continue;
        pl->list_host.push_back(c);
        pl->list_host.push_back(lfr::warp2_queue_dims(dim[c].e, dim[c].nc, dim[c].n2));
        g.bytes = std::max(g.bytes, b);
        ++g.n;
      }
      if (!g.n) continue;
      g.warps = pass == 0 ? W : std::min(W, kMaxSmemPerBlock / g.bytes);
      pl->launches.push_back(g);
    }
  }
  auto emit = [&](int r, const lfr_plan::SchedDim& d, int b, uint32_t offset, uint32_t n) {
    Launch L;
    L.kernel = fits_four(b) ? kFour[r] : kOne[r];
    L.offset = offset;
    L.n = n;
    L.emax = d.e;
    L.ncmax = d.nc;
    L.n2max = d.n2;
    L.bytes = b;
    L.warps = info(L.kernel).per_cta;
    pl->launches.push_back(L);
  };
  for (int k = n_class - 1; k >= 0; --k)
    for (int r = kRoutes - 1; r >= 0; --r) {
      const int key = r * n_class + k;
      const uint32_t n = count[key] - queued(key);
      if (!n) continue;
      if (bytes[key] <= kMaxSmemPerBlock) {
        emit(r, caps[key], bytes[key], start[key], n);
      } else {  // every member fits on its own but the union of their maxima does not: one launch each
        for (uint32_t i = 0; i < n; ++i) {
          const uint32_t c = pl->list_host[start[key] + i];
          emit(r, dim[c], slot_of(key, c), start[key] + i, 1);
        }
      }
    }
  return LFR_OK;
}

// CTA-tier components: the host only lays out per-component offsets (upper bounds: candidate edges
// from row_ptr, non-root nodes), in the order of the schedule's CTA launches, and sizes the HBM arrays;
// the kept-edge / in-edge lists, free-variable numbering and twins are built on the device by
// cta_prepare_kernel (launched by fill_plan once the edge records and local_of are in HBM).
int prepare_large(lfr_plan* pl, const lfr_problem* p, cudaStream_t s) {
  pl->n_large = (uint32_t)pl->large_slots.size();
  pl->L_total_free = 0;
  if (pl->n_large == 0) return LFR_OK;
  std::vector<lfr::CtaComp>& comps = pl->L_comps_host;  // plan member: the async upload reads it
  comps.assign(pl->n_large, lfr::CtaComp{});
  uint64_t e_off = 0, n_off = 0, f_off = 0, ell_off = 0, s_off = 0;
  for (uint32_t k = 0; k < pl->n_large; ++k) {
    const uint32_t c = pl->large_slots[k];
    const uint32_t nc = p->comp_ptr[c + 1] - p->comp_ptr[c];
    if (pl->large_cand[k] > 0xffffffffull) return fail(LFR_EUNSUPPORTED, "component with more than 2^32 out-edges");
    lfr::CtaComp& cc = comps[k];
    cc.slot = c;
    cc.Nc = nc;
    cc.Ec = 0;  // filled on the device, with nf and regular
    cc.nf = 0;
    cc.regular = 0;
    cc.e_off = e_off;
    cc.n_off = n_off;
    cc.f_off = f_off;
    cc.comp_index = k;
    cc.ell_off = ell_off;
    cc.s_off = s_off;
    ell_off += pl->large_ell[k];
    s_off += (nc + 31) / 32 + 1;
    e_off += pl->large_cand[k];
    n_off += nc;
    f_off += pl->large_free[k];
  }
  pl->L_total_free = f_off;
  const uint64_t E1 = std::max<uint64_t>(e_off, 1), N1 = std::max<uint64_t>(n_off, 1), F1 = std::max<uint64_t>(f_off, 1);
  const uint64_t L1 = std::max<uint64_t>(ell_off, 1), S1 = std::max<uint64_t>(s_off, 1);
  LFR_TRY(upload(&pl->L_comps, comps.data(), comps.size(), s));
  LFR_TRY(pl->L_rec.reserve(sizeof(float4) * 5 * E1));
  LFR_TRY(pl->L_meta.reserve(sizeof(uint32_t) * E1));
  LFR_TRY(pl->L_inlist.reserve(sizeof(uint32_t) * E1));
  LFR_TRY(pl->L_twin.reserve(sizeof(uint32_t) * E1));
  LFR_TRY(pl->L_fdst.reserve(sizeof(int32_t) * E1));
  LFR_TRY(pl->L_bE01.reserve(sizeof(double2) * L1));
  LFR_TRY(pl->L_bE23.reserve(sizeof(double2) * L1));
  LFR_TRY(pl->L_fdstE.reserve(sizeof(int32_t) * L1));
  LFR_TRY(pl->L_ell_base.reserve(sizeof(uint32_t) * S1));
  LFR_TRY(pl->L_node.reserve(sizeof(uint32_t) * N1));
  LFR_TRY(pl->L_outptr.reserve(sizeof(uint32_t) * (N1 + pl->n_large)));
  LFR_TRY(pl->L_inptr.reserve(sizeof(uint32_t) * (N1 + pl->n_large)));
  LFR_TRY(pl->L_freeof.reserve(sizeof(int32_t) * N1));
  LFR_TRY(pl->L_lof.reserve(sizeof(uint32_t) * F1));
  LFR_TRY(pl->L_scr.reserve(sizeof(double) * 7 * E1));
  LFR_TRY(pl->L_q.reserve(sizeof(double) * 2 * E1));
  LFR_TRY(pl->L_x.reserve(sizeof(double) * 2 * N1));
  LFR_TRY(pl->L_xc.reserve(sizeof(double) * 2 * N1));
  LFR_TRY(pl->L_vec.reserve(sizeof(double) * (2 * lfr::V_COUNT + 9) * F1));
  return LFR_OK;
}

// Device-side address of a page-locked (cudaHostAlloc / cudaHostRegister) host buffer, or nullptr
// when the memory is pageable (or not 16-byte aligned, which the 128-bit accesses need).
void* device_view_of_pinned(const void* host_ptr) {
  if (!host_ptr || (reinterpret_cast<uintptr_t>(host_ptr) & 15u)) return nullptr;
  cudaPointerAttributes a;
  if (cudaPointerGetAttributes(&a, host_ptr) != cudaSuccess) {
    cudaGetLastError();
    return nullptr;
  }
  if (a.type != cudaMemoryTypeHost || !a.devicePointer) return nullptr;
  return a.devicePointer;
}

int schedule_plan(lfr_plan* pl, const lfr_problem* p, cudaStream_t s);

// (Re)fill a plan from host arrays: H2D copies + schedule.  Buffers only grow.
// zc_edges / zc_positions: device-side views of the caller's pinned buffers (lfr_solve() only):
// the staging tiers then read the edge records / write the results there, and the 80-byte records
// — 95 % of the input bytes — are copied to HBM only if some non-staging tier needs them.
int fill_plan(lfr_plan* pl, const lfr_problem* p, const lfr_options& o, const double* initial_positions,
              cudaStream_t s, bool stage_positions_directly = false, const float4* zc_edges = nullptr,
              double* zc_positions = nullptr, bool graph_resident = false) {
  pl->opt = o;
  pl->K = make_consts(o);
  pl->N = p->n_nodes;
  pl->C = p->n_components;
  pl->E = p->n_edges;
  pl->total_slots = p->n_components ? p->comp_ptr[p->n_components] : 0;
  pl->profile = (o.debug_flags & LFR_DBG_PROFILE) != 0;
  pl->zc_edges = zc_edges;
  pl->zc_positions = zc_positions;
  // graph_resident: lfr_plan_create_from_matches() built the edge records and the six per-node / dispatch
  // arrays in the plan's buffers already; only the host copies in `p` are read (by the schedule builder)
  pl->edges_in_hbm = graph_resident;
  if (!zc_edges && !graph_resident) {
    LFR_TRY(upload(&pl->edges, p->edges, (size_t)p->n_edges, s));  // the bulk first: the DMA runs while the host schedules
    pl->edges_in_hbm = true;
  }
  // the small per-node arrays gate the first launch: with zero-copy edges they ARE the upload, so they
  // go out on two streams (two copy engines) instead of queueing behind each other
  cudaStream_t s2 = s;
  if (zc_edges) {
    if (!pl->copy_stream) LFR_CUDA(cudaStreamCreateWithFlags(&pl->copy_stream, cudaStreamNonBlocking));
    if (!pl->ev_small) LFR_CUDA(cudaEventCreateWithFlags(&pl->ev_small, cudaEventDisableTiming));
    s2 = pl->copy_stream;
    LFR_CUDA(cudaEventRecord(pl->ev_small, s));          // orders s2's copies after whatever `s` ran before
    LFR_CUDA(cudaStreamWaitEvent(s2, pl->ev_small, 0));
  }
  if (!graph_resident) {
    LFR_TRY(upload(&pl->row_ptr, p->row_ptr, (size_t)p->n_nodes + 1, s));
    LFR_TRY(upload(&pl->track, p->track, (size_t)p->n_nodes, s2));
    LFR_TRY(upload(&pl->comp, p->comp, (size_t)p->n_nodes, s2));
    LFR_TRY(upload(&pl->is_root, p->is_root, (size_t)p->n_nodes, s2));
    LFR_TRY(upload(&pl->comp_ptr, p->comp_ptr, (size_t)p->n_components + 1, s));
    LFR_TRY(upload(&pl->comp_nodes, p->comp_nodes, (size_t)pl->total_slots, s));
  }
  if (s2 != s) {
    LFR_CUDA(cudaEventRecord(pl->ev_small, s2));
    LFR_CUDA(cudaStreamWaitEvent(s, pl->ev_small, 0));
  }
  const size_t N = std::max<size_t>(pl->N, 1), C = std::max<size_t>(pl->C, 1);
  LFR_TRY(pl->local_of.reserve(sizeof(uint32_t) * N));
  LFR_TRY(pl->pos.reserve(sizeof(double) * 2 * N));
  pl->Cp = (uint32_t)((C + 1) & ~(size_t)1);
  LFR_TRY(pl->stats.reserve(pl->stats_bytes()));
  if (pl->profile) {
    LFR_TRY(pl->cycles.reserve(sizeof(unsigned long long) * 8 * C));
    LFR_TRY(pl->times.reserve(sizeof(unsigned long long) * 2 * C));
    LFR_CUDA(cudaMemsetAsync(pl->cycles.p, 0, sizeof(unsigned long long) * 8 * C, s));
    LFR_CUDA(cudaMemsetAsync(pl->times.p, 0, sizeof(unsigned long long) * 2 * C, s));
  }
  // per-slot stats default to "skipped" (size-1 components never run); also clears the error flag
  LFR_CUDA(cudaMemsetAsync(pl->stats.p, 0, pl->stats_bytes(), s));
  if (stage_positions_directly) {
    // lfr_solve(): the caller's start point goes straight into the working array
    if (pl->N)
      LFR_CUDA(cudaMemcpyAsync(pl->pos.p, initial_positions, sizeof(double) * 2 * (size_t)pl->N,
                               cudaMemcpyHostToDevice, s));
    pl->pos_is_staged = true;
  } else {
    LFR_TRY(pl->pos_init.reserve(sizeof(double) * 2 * N));
    if (initial_positions && pl->N)
      LFR_CUDA(cudaMemcpyAsync(pl->pos_init.p, initial_positions, sizeof(double) * 2 * (size_t)pl->N,
                               cudaMemcpyHostToDevice, s));
    else
      LFR_CUDA(cudaMemsetAsync(pl->pos_init.p, 0, sizeof(double) * 2 * N, s));
    pl->pos_is_staged = false;
  }
  return schedule_plan(pl, p, s);
}

// The schedule of a filled plan and what it sizes: the launch list, the CTA tier's layout and preparation,
// the streams.  `p` holds the host copies of the per-node and dispatch arrays (is_root: the mask the
// tiers read); the device arrays are the plan's.
int schedule_plan(lfr_plan* pl, const lfr_problem* p, cudaStream_t s) {
  const float4* zc_edges = pl->zc_edges;
  host_mark(0);
  LFR_TRY(build_schedule(pl, p));  // host work overlaps the copies above
  host_mark(1);
  bool needs_hbm_edges = false, has_queue = false;
  for (const Launch& L : pl->launches) {
    needs_hbm_edges = needs_hbm_edges || info(L.kernel).edges == Edges::kGlobal;
    has_queue = has_queue || L.kernel == Kernel::kQueue;
  }
  // Zero-copy and the CTA tier: its preparation kernel can pull the records it keeps straight from the
  // pinned array, but SM loads over PCIe are slower than the copy engine, so that pays only while
  // those components hold less than ~0.3 of the edges
  // (one device of a multi-device solve); otherwise the whole array goes to HBM on the copy stream.
  uint64_t cta_cand = 0;
  for (uint64_t e : pl->large_cand) cta_cand += e;
  pl->cta_from_hbm = zc_edges && 10 * cta_cand > 3 * (uint64_t)p->n_edges;
  if (zc_edges && (needs_hbm_edges || pl->cta_from_hbm)) {
    // mixed schedule: the Cholesky-warp tier reads edge records from global memory by index, so the
    // array goes to HBM after all — on its own stream, and only that tier waits for it
    if (!pl->copy_stream) LFR_CUDA(cudaStreamCreateWithFlags(&pl->copy_stream, cudaStreamNonBlocking));
    if (!pl->ev_edges) LFR_CUDA(cudaEventCreateWithFlags(&pl->ev_edges, cudaEventDisableTiming));
    LFR_TRY(upload(&pl->edges, p->edges, (size_t)p->n_edges, pl->copy_stream));
    LFR_CUDA(cudaEventRecord(pl->ev_edges, pl->copy_stream));
    pl->edges_in_hbm = true;
  }
  LFR_TRY(prepare_large(pl, p, s));
  LFR_TRY(upload(&pl->lists, pl->list_host.data(), pl->list_host.size(), s));
  if (pl->total_slots) {
    lfr::local_index_kernel<<<(pl->total_slots + 255) / 256, 256, 0, s>>>(
        pl->comp_ptr.as<uint32_t>(), pl->comp_nodes.as<uint32_t>(), pl->C, pl->total_slots,
        pl->local_of.as<uint32_t>());
    LFR_CUDA(cudaGetLastError());
  }
  if (pl->n_large) {
    // kept-edge records / in-edge lists, free-variable numbering and twins of the CTA-tier components,
    // built on the device; with zero-copy edges the kernel either pulls exactly the records these
    // components keep from the caller's pinned array, or reads the bulk copy (see above)
    lfr::DevProblem P = pl->dev();
    cudaStream_t ps = s;
    if (zc_edges && !pl->cta_from_hbm) {
      P.edges = zc_edges;
    } else if (zc_edges) {
      // behind the bulk copy on the copy stream, once the small arrays and local_of (stream s) are
      // there; the CTA-tier launches wait for ev_edges, the staging tiers do not
      if (!pl->ev_prep) LFR_CUDA(cudaEventCreateWithFlags(&pl->ev_prep, cudaEventDisableTiming));
      LFR_CUDA(cudaEventRecord(pl->ev_prep, s));
      LFR_CUDA(cudaStreamWaitEvent(pl->copy_stream, pl->ev_prep, 0));
      ps = pl->copy_stream;
    }
    lfr::cta_prepare_kernel<<<pl->n_large, lfr::kCtaThreads, 0, ps>>>(P, pl->cta_arrays(), pl->L_comps.as<lfr::CtaComp>());
    LFR_CUDA(cudaGetLastError());
    if (ps != s) LFR_CUDA(cudaEventRecord(pl->ev_edges, pl->copy_stream));
  }
  // streams for concurrent bucket launches
  if (has_queue && !pl->queue_ctr.p) {
    // zero once: every queue launch leaves its two words at zero when it ends
    LFR_TRY(pl->queue_ctr.reserve(2 * sizeof(uint32_t) * 2));
    LFR_CUDA(cudaMemsetAsync(pl->queue_ctr.p, 0, pl->queue_ctr.cap, s));
  }
  if (has_queue && !pl->n_sms) LFR_CUDA(cudaDeviceGetAttribute(&pl->n_sms, cudaDevAttrMultiProcessorCount, pl->device));
  const int want = std::min<int>(kMaxStreams, std::max<int>(0, pl->num_launches() - 1));
  if (!pl->ev_fork) LFR_CUDA(cudaEventCreateWithFlags(&pl->ev_fork, cudaEventDisableTiming));
  while (pl->n_streams < want) {
    LFR_CUDA(cudaStreamCreateWithFlags(&pl->streams[pl->n_streams], cudaStreamNonBlocking));
    LFR_CUDA(cudaEventCreateWithFlags(&pl->ev_join[pl->n_streams], cudaEventDisableTiming));
    ++pl->n_streams;
  }
  return LFR_OK;
}

// Bytes of zero-copy staging pulls kept outstanding per device (stage_edges): large enough to cover
// the PCIe bandwidth-delay product, small enough that records arrive in dispatch order.
// LFR_PULL_WINDOW_KB overrides (0 = unpaced), read once.
unsigned zero_copy_pull_window() {
  static const unsigned w = [] {
    const char* e = std::getenv("LFR_PULL_WINDOW_KB");
    if (e && *e) return (unsigned)std::strtoul(e, nullptr, 10) * 1024u;
    return 512u * 1024u;
  }();
  return w;
}

// ---- the graph stage on the device (include/lfr_graph.h, lfr_graph.cuh) ----------------------------
struct TmpBuf : DevBuf {
  ~TmpBuf() { release(); }
};

inline unsigned blocks_for(uint64_t n) { return (unsigned)((n + 255) / 256); }

int bits_for(uint64_t max_value) {  // radix-sort key width that covers 0..max_value
  int b = 1;
  while (b < 64 && (max_value >> b)) ++b;
  return b;
}

struct MaxOp {
  __device__ __forceinline__ uint32_t operator()(uint32_t a, uint32_t b) const { return a > b ? a : b; }
};

// The calling thread's device operations since lfr_debug_device_ops() last reset them: {kernel launch sites checked,
// CUB calls, synchronising copies to the host} (a test hook: a call's count must not grow with its input's groups)
thread_local unsigned long long g_device_ops[3] = {};

// one CUB device call: size query, temporary storage, run
template <typename F>
int cub_run(DevBuf& tmp, F&& f) {
  ++g_device_ops[1];
  size_t bytes = 0;
  LFR_CUDA(f(static_cast<void*>(nullptr), bytes));
  LFR_TRY(tmp.reserve(std::max<size_t>(bytes, 1)));
  LFR_CUDA(f(tmp.p, bytes));
  return LFR_OK;
}

template <typename T>
int fetch(T* h, const void* d, size_t count, cudaStream_t s) {
  if (!count) return LFR_OK;
  ++g_device_ops[2];
  LFR_CUDA(cudaMemcpyAsync(h, d, count * sizeof(T), cudaMemcpyDeviceToHost, s));
  LFR_CUDA(cudaStreamSynchronize(s));
  return LFR_OK;
}

#define LFR_LAUNCHED()  \
  do {                   \
    ++g_device_ops[0];   \
    LFR_CUDA(cudaGetLastError()); \
  } while (0)

// Connected components of 0..n-1 over the edges (a[i], b[i]) (only those inside one group of `gc`
// when given), labelled in order of their lowest member: label[n], returns the count in *n_out.
int components_on_device(uint32_t n, const uint32_t* a, const uint32_t* b, uint32_t m, const uint32_t* gc, uint32_t* label,
                         uint32_t* n_out, DevBuf& tmp, cudaStream_t s) {
  TmpBuf par, rep, lab;
  LFR_TRY(par.reserve(4 * (size_t)n));
  LFR_TRY(rep.reserve(4 * ((size_t)n + 1)));
  LFR_TRY(lab.reserve(4 * ((size_t)n + 1)));
  lfr::graph::iota_kernel<<<blocks_for(n), 256, 0, s>>>(par.as<uint32_t>(), n);
  if (m) lfr::graph::cc_hook_kernel<<<blocks_for(m), 256, 0, s>>>(a, b, m, gc, par.as<uint32_t>());
  lfr::graph::cc_flatten_kernel<<<blocks_for(n), 256, 0, s>>>(par.as<uint32_t>(), n, rep.as<uint32_t>());
  LFR_LAUNCHED();
  LFR_CUDA(cudaMemsetAsync(rep.as<uint32_t>() + n, 0, 4, s));
  uint32_t* rp = rep.as<uint32_t>();
  uint32_t* lp = lab.as<uint32_t>();
  LFR_TRY(cub_run(tmp, [&](void* t, size_t& nb) { return cub::DeviceScan::ExclusiveSum(t, nb, rp, lp, (int)n + 1, s); }));
  lfr::graph::cc_label_kernel<<<blocks_for(n), 256, 0, s>>>(par.as<uint32_t>(), lp, n, label);
  LFR_LAUNCHED();
  return fetch(n_out, lp + n, 1, s);
}

// ---- the recursive cut on the device (lfr_cut.cuh) --------------------------------------------------
// undirected edges of one recursion level, grouped by sub-problem (sub ascending)
struct CutLists {
  TmpBuf a, b, w, sub;
  int reserve(size_t m) {
    m = std::max<size_t>(m, 1);
    LFR_TRY(a.reserve(4 * m));
    LFR_TRY(b.reserve(4 * m));
    LFR_TRY(w.reserve(8 * m));
    LFR_TRY(sub.reserve(4 * m));
    return LFR_OK;
  }
};

struct SumLL {
  __device__ __forceinline__ long long operator()(long long a, long long b) const { return a + b; }
};

// The edges idx[0..n) of `src` into `dst`, grouped by key (key_bits wide): the sub-problem of an edge is
// the rank of its key.  `key` is overwritten.
int group_cut_edges(uint32_t* key, const uint32_t* idx, uint32_t n, int key_bits, CutLists& src, CutLists& dst, uint32_t* n_sub,
                    DevBuf& tmp, cudaStream_t s) {
  TmpBuf k2, i2, head;
  LFR_TRY(k2.reserve(4 * (size_t)n));
  LFR_TRY(i2.reserve(4 * (size_t)n));
  LFR_TRY(head.reserve(4 * (size_t)n));
  uint32_t *kk = k2.as<uint32_t>(), *ii = i2.as<uint32_t>(), *h = head.as<uint32_t>();
  LFR_TRY(cub_run(tmp, [&](void* t, size_t& nb) { return cub::DeviceRadixSort::SortPairs(t, nb, key, kk, idx, ii, (int)n, 0, key_bits, s); }));
  lfr::cut::heads_kernel<<<blocks_for(n), 256, 0, s>>>(kk, n, h);
  LFR_LAUNCHED();
  LFR_TRY(cub_run(tmp, [&](void* t, size_t& nb) { return cub::DeviceScan::InclusiveSum(t, nb, h, key, (int)n, s); }));
  lfr::cut::gather_edges_kernel<<<blocks_for(n), 256, 0, s>>>(ii, key, n, src.a.as<uint32_t>(), src.b.as<uint32_t>(), src.w.as<long long>(),
                                                              dst.a.as<uint32_t>(), dst.b.as<uint32_t>(), dst.w.as<long long>(),
                                                              dst.sub.as<uint32_t>());
  LFR_LAUNCHED();
  return fetch(n_sub, key + n - 1, 1, s);
}

// lfr_cut.h recursive_cut_all on the device, one launch set per recursion level.  E[0] holds the roots'
// m edges (no self-loops) over nodes 0..n_nodes-1, grouped into n_sub roots; E[1] has room for m edges.
// Every node of a root gets label[x] = label_base + (the lowest node of its group); *n_groups = groups.
// node_cap (device, may be NULL): a per-node max_weight, the same for every node of a root (sub-scenes).
int recursive_cut_on_device(uint32_t n_nodes, CutLists (&E)[2], uint32_t m, uint32_t n_sub, const uint32_t* node_weight,
                            uint64_t max_weight, uint32_t label_base, uint32_t* label, uint32_t* n_groups, DevBuf& tmp, cudaStream_t s,
                            const uint32_t* node_cap = nullptr) {
  using namespace lfr::cut;
  *n_groups = 0;
  if (!m) return LFR_OK;
  const size_t N = n_nodes, H = 2 * (size_t)m, NL = std::min(N, H);
  TmpBuf beg, end, vol, vis, claim, side, sub_of, covered;                        // per node
  TmpBuf hk, hk2, hw, hw2, uk, uw, nbr, head, hnode, hsub, lnode, lsub, lnode2, lsub2;  // per half-edge
  TmpBuf order, pstart, pvol, pidx, pside;                                        // per node of the level
  TmpBuf node_ptr, side_w, side_min, cont;                                        // per sub-problem
  TmpBuf keep, key, iota, kidx, kkey, cnt;                                        // per edge
  for (TmpBuf* b : {&beg, &end, &vis, &claim, &sub_of, &covered}) LFR_TRY(b->reserve(4 * N));
  LFR_TRY(vol.reserve(8 * N));
  LFR_TRY(side.reserve(N));
  for (TmpBuf* b : {&hk, &hk2, &hw, &hw2, &uk, &uw}) LFR_TRY(b->reserve(8 * H));
  for (TmpBuf* b : {&nbr, &head, &hnode, &hsub, &lnode, &lsub, &lnode2, &lsub2}) LFR_TRY(b->reserve(4 * H));
  for (TmpBuf* b : {&order, &pstart, &pidx}) LFR_TRY(b->reserve(4 * NL));
  LFR_TRY(pvol.reserve(8 * NL));
  LFR_TRY(pside.reserve(NL));
  LFR_TRY(node_ptr.reserve(4 * ((size_t)m + 1)));
  LFR_TRY(side_w.reserve(16 * (size_t)m));
  LFR_TRY(side_min.reserve(8 * (size_t)m));
  LFR_TRY(cont.reserve(2 * (size_t)m));
  for (TmpBuf* b : {&keep, &key, &iota, &kidx, &kkey}) LFR_TRY(b->reserve(4 * (size_t)m));
  LFR_TRY(cnt.reserve(16));
  LFR_CUDA(cudaMemsetAsync(vis.p, 0, 4 * N, s));
  LFR_CUDA(cudaMemsetAsync(covered.p, 0, 4 * N, s));
  LFR_CUDA(cudaMemsetAsync(cnt.p, 0, 16, s));
  uint32_t* d_groups = cnt.as<uint32_t>();
  uint32_t* d_count = d_groups + 1;
  const int bits = bits_for(std::max<uint32_t>(n_nodes, 2) - 1);
  int cur = 0;
  for (uint32_t lvl = 0;; ++lvl) {
    CutLists& C = E[cur];
    half_edges_kernel<<<blocks_for(m), 256, 0, s>>>(C.a.as<uint32_t>(), C.b.as<uint32_t>(), C.w.as<long long>(), C.sub.as<uint32_t>(), m,
                                                    bits, hk.as<unsigned long long>(), hw.as<long long>(), sub_of.as<uint32_t>());
    LFR_LAUNCHED();
    {
      unsigned long long *k1 = hk.as<unsigned long long>(), *k2 = hk2.as<unsigned long long>(), *ku = uk.as<unsigned long long>();
      long long *w1 = hw.as<long long>(), *w2 = hw2.as<long long>(), *wu = uw.as<long long>();
      const int nh = (int)(2 * m);
      LFR_TRY(cub_run(tmp, [&](void* t, size_t& nb) { return cub::DeviceRadixSort::SortPairs(t, nb, k1, k2, w1, w2, nh, 0, 2 * bits, s); }));
      LFR_TRY(cub_run(tmp, [&](void* t, size_t& nb) {
        return cub::DeviceReduce::ReduceByKey(t, nb, k2, ku, w2, wu, d_count, SumLL(), nh, s);
      }));
    }
    rows_kernel<<<blocks_for(2 * (uint64_t)m), 256, 0, s>>>(uk.as<unsigned long long>(), d_count, 2 * m, bits, sub_of.as<uint32_t>(),
                                                            nbr.as<uint32_t>(), beg.as<uint32_t>(), end.as<uint32_t>(), head.as<uint32_t>(),
                                                            hnode.as<uint32_t>(), hsub.as<uint32_t>());
    LFR_LAUNCHED();
    uint32_t n_lev = 0;
    {
      uint32_t *h = head.as<uint32_t>(), *hn = hnode.as<uint32_t>(), *hs = hsub.as<uint32_t>(), *ln = lnode.as<uint32_t>(),
               *ls = lsub.as<uint32_t>(), *c = d_count + 1;
      const int nh = (int)(2 * m);
      LFR_TRY(cub_run(tmp, [&](void* t, size_t& nb) { return cub::DeviceSelect::Flagged(t, nb, hn, h, ln, c, nh, s); }));
      LFR_TRY(cub_run(tmp, [&](void* t, size_t& nb) { return cub::DeviceSelect::Flagged(t, nb, hs, h, ls, c, nh, s); }));
      LFR_TRY(fetch(&n_lev, c, 1, s));
      uint32_t *ln2 = lnode2.as<uint32_t>(), *ls2 = lsub2.as<uint32_t>();
      LFR_TRY(cub_run(tmp, [&](void* t, size_t& nb) {
        return cub::DeviceRadixSort::SortPairs(t, nb, ls, ls2, ln, ln2, (int)n_lev, 0, bits_for(std::max<uint32_t>(n_sub, 2) - 1), s);
      }));
    }
    node_ptr_kernel<<<blocks_for(n_lev), 256, 0, s>>>(lsub2.as<uint32_t>(), n_lev, n_sub, node_ptr.as<uint32_t>());
    LFR_LAUNCHED();
    Level L;
    L.nodes = lnode2.as<uint32_t>();
    L.node_ptr = node_ptr.as<uint32_t>();
    L.beg = beg.as<uint32_t>();
    L.end = end.as<uint32_t>();
    L.nbr = nbr.as<uint32_t>();
    L.w = uw.as<long long>();
    L.node_weight = node_weight;
    L.vol = vol.as<long long>();
    L.vis = vis.as<uint32_t>();
    L.claim = claim.as<uint32_t>();
    L.side = side.as<uint8_t>();
    L.order = order.as<uint32_t>();
    L.piece_start = pstart.as<uint32_t>();
    L.pvol = pvol.as<long long>();
    L.pidx = pidx.as<uint32_t>();
    L.pside = pside.as<uint8_t>();
    L.stamp = 2 * lvl + 1;
    L.max_weight = max_weight;
    L.node_cap = node_cap;
    L.side_w = side_w.as<long long>();
    L.side_min = side_min.as<uint32_t>();
    L.cont = cont.as<uint8_t>();
    L.n_groups = d_groups;
    cut_sub_kernel<<<n_sub, kThreads, 0, s>>>(L);
    keep_edges_kernel<<<blocks_for(m), 256, 0, s>>>(C.a.as<uint32_t>(), C.b.as<uint32_t>(), C.sub.as<uint32_t>(), m, side.as<uint8_t>(),
                                                    cont.as<uint8_t>(), lvl + 1, covered.as<uint32_t>(), keep.as<uint32_t>(),
                                                    key.as<uint32_t>());
    label_nodes_kernel<<<blocks_for(n_lev), 256, 0, s>>>(lnode2.as<uint32_t>(), lsub2.as<uint32_t>(), n_lev, side.as<uint8_t>(),
                                                         cont.as<uint8_t>(), side_min.as<uint32_t>(), covered.as<uint32_t>(), lvl + 1,
                                                         label_base, label, d_groups);
    lfr::graph::iota_kernel<<<blocks_for(m), 256, 0, s>>>(iota.as<uint32_t>(), m);
    LFR_LAUNCHED();
    uint32_t m2 = 0;
    {
      uint32_t *fl = keep.as<uint32_t>(), *io = iota.as<uint32_t>(), *ki = kidx.as<uint32_t>(), *ky = key.as<uint32_t>(),
               *kk = kkey.as<uint32_t>(), *c = d_count + 2;
      LFR_TRY(cub_run(tmp, [&](void* t, size_t& nb) { return cub::DeviceSelect::Flagged(t, nb, io, fl, ki, c, (int)m, s); }));
      LFR_TRY(cub_run(tmp, [&](void* t, size_t& nb) { return cub::DeviceSelect::Flagged(t, nb, ky, fl, kk, c, (int)m, s); }));
      LFR_TRY(fetch(&m2, c, 1, s));
    }
    if (!m2) break;
    uint32_t n_sub2 = 0;
    LFR_TRY(group_cut_edges(kkey.as<uint32_t>(), kidx.as<uint32_t>(), m2, bits_for(2 * (uint64_t)n_sub - 1), C, E[1 - cur], &n_sub2, tmp, s));
    // every edge kept and one child per sub-problem: every sub-problem put all its nodes on one side (its
    // pieces all have volume <= 0), and lfr_cut.h would cut it again forever
    if (m2 == m && n_sub2 == n_sub) return fail(LFR_EINVAL, "recursive cut makes no progress (meta-edge weights <= 0)");
    cur = 1 - cur;
    m = m2;
    n_sub = n_sub2;
  }
  return fetch(n_groups, d_groups, 1, s);
}

using Clock = std::chrono::steady_clock;
double ms_since(Clock::time_point t0) { return std::chrono::duration<double, std::milli>(Clock::now() - t0).count(); }

// lfr_graph_stage_on_device(): the directed edges from which the graph stage runs on the device.  The
// native drop-in's "Total time" on an H100 80GB HBM3 at 700 W (tools/gpu_graph_stage_time.py, DESIGN.md
// §4): the host route is faster up to ~10 K directed edges and the device route from 200 K on; in between
// the two trade places from run to run within their spread, and the switch sits inside that tie.
constexpr uint64_t kDeviceGraphStageMinEdges = 32768;
// lfr_wire_decode_on_device(): the matches from which the drop-in decodes them on the device.  On an
// H100 80GB HBM3 (tools/gpu_wire_decode_time.py, DESIGN.md §4) lfr_plan_create_from_wire() alone beats the
// host decode + lfr_plan_create_from_matches() from 100 K matches on, but the drop-in's host decode runs
// while CUDA starts up: its wall time gains from 634 K matches (cfg4) on and ties at 100-137 K.
constexpr uint64_t kDeviceDecodeMinMatches = 262144;
// lfr_last_error() of lfr_plan_create_from_wire() on a malformed Match (include/lfr_graph.h)
constexpr const char* kMalformedMatch = "malformed Match message";

// The graph stage's input on the device: feat1 / feat2 / sim [n_matches], disp1 / disp2 [18 n_matches],
// match k of every pair at its global index (the order of lfr_host_input).
struct MatchArrays {
  TmpBuf feat1, feat2, sim, disp1, disp2;
};

// lfr_host_stage_create() on the device, block for block (lfr_host.cc), from the pair level of `in` and the
// device-resident matches `d` (in->feat1 ... in->disp2 are not read): the edge records go into pl->edges,
// the other arrays come back to pl->graph (the schedule builder is host code and reads them).
// device_cut (LFR_DBG_DEVICE_CUT): oversized meta-components are cut on the device (lfr_cut.cuh, the same
// groups) instead of by lfr_cut.h on host threads.  It is not the default: on an H100 80GB HBM3 at 700 W the
// device cut was slower than the host cut on every workload from cfg2 to cfg5 (tools/gpu_graph_cut_time.py,
// DESIGN.md §4), so no input size selects it.
int build_graph_on_device(const lfr_host_input* in, MatchArrays& d, lfr_plan* pl, lfr_host_sizes* S, bool device_cut,
                          cudaStream_t s) {
  using namespace lfr::graph;
  std::memset(S, 0, sizeof *S);
  auto G = std::make_unique<lfr_plan::GraphArrays>();
  const uint64_t P = in->n_pairs;
  const uint32_t n_images = in->n_images;
  // sub-scenes (lfr_host_input::image_group): each image's index inside its sub-scene and the set width, as
  // lfr_host.cc has them; the cut cap of each image's sub-scene once the seen images are known
  const uint32_t* group = in->image_group;
  std::vector<uint32_t> local_image, image_cap;
  uint32_t set_width = n_images, n_groups = 0;
  if (group) {
    for (uint32_t i = 0; i < n_images; ++i) n_groups = std::max(n_groups, group[i] + 1);
    std::vector<uint32_t> n_in_group(n_groups, 0);
    local_image.resize(n_images);
    for (uint32_t i = 0; i < n_images; ++i) local_image[i] = n_in_group[group[i]]++;
    set_width = n_groups ? *std::max_element(n_in_group.begin(), n_in_group.end()) : 0;
    for (uint64_t p = 0; p < in->n_pairs; ++p)  // a pair spans two sub-scenes: the host stage's LFR_EINVAL
      if (!(in->pair_skip && in->pair_skip[p]) && in->pair_img1[p] < n_images && in->pair_img2[p] < n_images &&
          group[in->pair_img1[p]] != group[in->pair_img2[p]])
        return fail(LFR_EINVAL, "a pair spans two sub-scenes");
  }
  TmpBuf tmp, d_img1, d_img2, d_skip, d_ptr, d_cnt, d_off, d_seen, d_err;
  const auto t_graph = Clock::now();
  // ---- H1: the match list -------------------------------------------------------------------------
  uint64_t M = 0;
  if (P) {
    LFR_TRY(upload(&d_img1, in->pair_img1, P, s));
    LFR_TRY(upload(&d_img2, in->pair_img2, P, s));
    if (in->pair_skip) LFR_TRY(upload(&d_skip, in->pair_skip, P, s));
    LFR_TRY(upload(&d_ptr, in->pair_ptr, P + 1, s));
    LFR_TRY(d_cnt.reserve(8 * (P + 1)));
    LFR_TRY(d_off.reserve(8 * (P + 1)));
    LFR_TRY(d_seen.reserve(std::max<size_t>(n_images, 1)));
    LFR_TRY(d_err.reserve(8));
    LFR_CUDA(cudaMemsetAsync(d_cnt.p, 0, 8 * (P + 1), s));
    LFR_CUDA(cudaMemsetAsync(d_seen.p, 0, std::max<size_t>(n_images, 1), s));
    LFR_CUDA(cudaMemsetAsync(d_err.p, 0, 8, s));
    pair_count_kernel<<<blocks_for(P), 256, 0, s>>>(d_img1.as<uint32_t>(), d_img2.as<uint32_t>(),
                                                    in->pair_skip ? d_skip.as<uint8_t>() : nullptr, d_ptr.as<uint64_t>(), P,
                                                    n_images, d_cnt.as<uint64_t>(), d_seen.as<uint8_t>(), d_err.as<int>());
    LFR_LAUNCHED();
    uint64_t* cp = d_cnt.as<uint64_t>();
    uint64_t* op = d_off.as<uint64_t>();
    if (P + 1 >= (1ull << 31)) return fail(LFR_EUNSUPPORTED, "more than 2^31 - 2 pairs");
    LFR_TRY(cub_run(tmp, [&](void* t, size_t& nb) { return cub::DeviceScan::ExclusiveSum(t, nb, cp, op, (int)(P + 1), s); }));
    int err[2];
    LFR_TRY(fetch(err, d_err.p, 2, s));
    if (err[0]) return fail(LFR_EINVAL, "image id out of range");
    LFR_TRY(fetch(&M, op + P, 1, s));
    std::vector<uint8_t> seen(n_images);
    LFR_TRY(fetch(seen.data(), d_seen.p, n_images, s));
    for (uint8_t v : seen) S->n_images_seen += v;
    if (group) {
      std::vector<uint32_t> group_seen(n_groups, 0);
      for (uint32_t i = 0; i < n_images; ++i) group_seen[group[i]] += seen[i];
      image_cap.resize(n_images);
      for (uint32_t i = 0; i < n_images; ++i) image_cap[i] = group_seen[group[i]];
    }
  }
  if (2 * M >= (1ull << 31)) return fail(LFR_EUNSUPPORTED, "more than 2^31 - 1 directed edges");
  const uint64_t E = 2 * M;
  TmpBuf d_kept, d_key, d_key2, d_pos, d_pos2, d_first, d_id, d_head, d_headof, d_nop;
  uint32_t N = 0;
  if (M) {
    LFR_TRY(d_kept.reserve(8 * M));
    LFR_TRY(d_key.reserve(8 * E));
    LFR_TRY(d_key2.reserve(8 * E));
    LFR_TRY(d_pos.reserve(4 * E));
    LFR_TRY(d_pos2.reserve(4 * E));
    expand_matches_kernel<<<blocks_for(M), 256, 0, s>>>(d_off.as<uint64_t>(), P, d_img1.as<uint32_t>(), d_img2.as<uint32_t>(),
                                                        d_ptr.as<uint64_t>(), d.feat1.as<uint32_t>(), d.feat2.as<uint32_t>(),
                                                        d.sim.as<float>(), M, d_kept.as<uint64_t>(),
                                                        d_key.as<unsigned long long>(), d_pos.as<uint32_t>(), d_err.as<int>());
    LFR_LAUNCHED();
    int err[2];
    LFR_TRY(fetch(err, d_err.p, 2, s));
    if (err[1]) return fail(LFR_EINVAL, "non-finite similarity");
    // (image, feature) -> node id in order of first appearance: stable sort of (key, position); the
    // first position of every key gets the next id in position order
    {
      unsigned long long *k1 = d_key.as<unsigned long long>(), *k2 = d_key2.as<unsigned long long>();
      uint32_t *p1 = d_pos.as<uint32_t>(), *p2 = d_pos2.as<uint32_t>();
      const int end_bit = 32 + bits_for(n_images);
      LFR_TRY(cub_run(tmp, [&](void* t, size_t& nb) {
        return cub::DeviceRadixSort::SortPairs(t, nb, k1, k2, p1, p2, (int)E, 0, end_bit, s);
      }));
    }
    LFR_TRY(d_first.reserve(4 * E));
    LFR_TRY(d_id.reserve(4 * E));
    LFR_TRY(d_head.reserve(4 * E));
    LFR_TRY(d_headof.reserve(4 * E));
    first_flags_kernel<<<blocks_for(E), 256, 0, s>>>(d_key2.as<unsigned long long>(), d_pos2.as<uint32_t>(), E,
                                                     d_first.as<uint32_t>(), d_head.as<uint32_t>());
    LFR_LAUNCHED();
    {
      uint32_t *f = d_first.as<uint32_t>(), *id = d_id.as<uint32_t>(), *h = d_head.as<uint32_t>(), *ho = d_headof.as<uint32_t>();
      LFR_TRY(cub_run(tmp, [&](void* t, size_t& nb) { return cub::DeviceScan::ExclusiveSum(t, nb, f, id, (int)E, s); }));
      LFR_TRY(cub_run(tmp, [&](void* t, size_t& nb) { return cub::DeviceScan::InclusiveScan(t, nb, h, ho, MaxOp(), (int)E, s); }));
      uint32_t last[2];
      LFR_TRY(fetch(&last[0], id + E - 1, 1, s));
      LFR_TRY(fetch(&last[1], f + E - 1, 1, s));
      N = last[0] + last[1];
    }
  }
  pl->graph.reset();
  if (N == 0) {
    G->row_ptr.assign(1, 0);
    G->comp_ptr.assign(1, 0);
    pl->graph = std::move(G);
    return LFR_OK;
  }
  if (n_images > 65535) return fail(LFR_EUNSUPPORTED, "more than 65535 images");
  TmpBuf d_ssrc, d_perm, d_cdst, d_csim;
  // the six arrays fill_plan() would upload are built in the plan's own buffers and stay there, and so do
  // the node -> (image, feature) ids, which lfr_plan_encode_solution() reads
  DevBuf &d_rowptr = pl->row_ptr, &d_track = pl->track, &d_isroot = pl->is_root, &d_comp = pl->comp,
         &d_cptr = pl->comp_ptr, &d_cnodes = pl->comp_nodes, &d_nimg = pl->node_image, &d_nfeat = pl->node_feat;
  LFR_TRY(d_nop.reserve(4 * E));
  LFR_TRY(d_nimg.reserve(4 * (size_t)N));
  LFR_TRY(d_nfeat.reserve(4 * (size_t)N));
  assign_nodes_kernel<<<blocks_for(E), 256, 0, s>>>(d_key2.as<unsigned long long>(), d_pos2.as<uint32_t>(), d_headof.as<uint32_t>(),
                                                    d_id.as<uint32_t>(), E, d_nop.as<uint32_t>(), d_nimg.as<uint32_t>(),
                                                    d_nfeat.as<uint32_t>());
  LFR_LAUNCHED();
  // CSR: a stable sort of the directed edges (position j = 2k + side) by source keeps add_edge order
  LFR_TRY(d_ssrc.reserve(4 * E));
  LFR_TRY(d_perm.reserve(4 * E));
  {
    uint32_t* iota = d_pos.as<uint32_t>();
    iota_kernel<<<blocks_for(E), 256, 0, s>>>(iota, E);
    LFR_LAUNCHED();
    uint32_t *src = d_nop.as<uint32_t>(), *ssrc = d_ssrc.as<uint32_t>(), *perm = d_perm.as<uint32_t>();
    const int end_bit = bits_for(N);
    LFR_TRY(cub_run(tmp, [&](void* t, size_t& nb) {
      return cub::DeviceRadixSort::SortPairs(t, nb, src, ssrc, iota, perm, (int)E, 0, end_bit, s);
    }));
  }
  LFR_TRY(d_rowptr.reserve(4 * ((size_t)N + 1)));
  row_ptr_kernel<<<blocks_for(E), 256, 0, s>>>(d_ssrc.as<uint32_t>(), E, N, d_rowptr.as<uint32_t>());
  LFR_TRY(pl->edges.reserve(sizeof(lfr_edge) * E));
  LFR_TRY(d_cdst.reserve(4 * E));
  LFR_TRY(d_csim.reserve(4 * E));
  edge_records_kernel<<<blocks_for(E), 256, 0, s>>>(d_perm.as<uint32_t>(), E, d_kept.as<uint64_t>(), d_nop.as<uint32_t>(),
                                                    d.sim.as<float>(), d.disp1.as<float>(), d.disp2.as<float>(),
                                                    pl->edges.as<lfr_edge>(), d_cdst.as<uint32_t>(), d_csim.as<float>());
  LFR_LAUNCHED();
  d.disp1.release();
  d.disp2.release();
  LFR_CUDA(cudaStreamSynchronize(s));
  S->graph_ms = ms_since(t_graph);
  const auto t_tracks = Clock::now();
  // ---- H2: constrained Kruskal: the sequential loop's order is descending (sim, n1, n2, k) ------------
  TmpBuf d_order, d_parent, d_size, d_res, d_mask, d_lists, d_slot, d_pool, d_pool_next;
  LFR_TRY(d_order.reserve(4 * M));
  {
    uint32_t *iota = d_pos.as<uint32_t>(), *n2k = d_first.as<uint32_t>(), *n2s = d_head.as<uint32_t>(), *perm1 = d_id.as<uint32_t>();
    iota_kernel<<<blocks_for(M), 256, 0, s>>>(iota, M);
    kruskal_keys_kernel<<<blocks_for(M), 256, 0, s>>>(d_nop.as<uint32_t>(), M, n2k);
    LFR_LAUNCHED();
    const int nb1 = bits_for(N);
    LFR_TRY(cub_run(tmp, [&](void* t, size_t& nb) {
      return cub::DeviceRadixSort::SortPairs(t, nb, n2k, n2s, iota, perm1, (int)M, 0, nb1, s);
    }));
    unsigned long long *k1 = d_key.as<unsigned long long>(), *k2 = d_key2.as<unsigned long long>();
    kruskal_keys2_kernel<<<blocks_for(M), 256, 0, s>>>(perm1, d_kept.as<uint64_t>(), d_nop.as<uint32_t>(), d.sim.as<float>(), M, nb1, k1);
    LFR_LAUNCHED();
    uint32_t* ord = d_order.as<uint32_t>();
    LFR_TRY(cub_run(tmp, [&](void* t, size_t& nb) {
      return cub::DeviceRadixSort::SortPairs(t, nb, k1, k2, perm1, ord, (int)M, 0, 32 + nb1, s);
    }));
  }
  UfState U;
  std::memset(&U, 0, sizeof U);
  U.small_sets = set_width <= 64;
  U.W = (set_width + 63) / 64;
  LFR_TRY(d_parent.reserve(4 * (size_t)N));
  LFR_TRY(d_size.reserve(4 * (size_t)N));
  LFR_TRY(d_res.reserve(4 * (size_t)N));
  U.parent = d_parent.as<int32_t>();
  U.size = d_size.as<uint32_t>();
  U.res = d_res.as<uint32_t>();
  U.node_image = d_nimg.as<uint32_t>();
  TmpBuf d_local, d_nloc;
  if (group) {  // the sets index images inside their sub-scene
    LFR_TRY(upload(&d_local, local_image.data(), n_images, s));
    LFR_TRY(d_nloc.reserve(4 * (size_t)N));
    gather_kernel<<<blocks_for(N), 256, 0, s>>>(d_nimg.as<uint32_t>(), d_local.as<uint32_t>(), N, d_nloc.as<uint32_t>());
    LFR_LAUNCHED();
    U.node_image = d_nloc.as<uint32_t>();
  }
  if (U.small_sets) {
    LFR_TRY(d_mask.reserve(8 * (size_t)N));
    U.mask = d_mask.as<unsigned long long>();
  } else {
    // a set crosses kListMax at most N / (kListMax + 1) times, and only then takes a bitset
    const size_t slots = (size_t)N / (kListMax + 1) + 1;
    LFR_TRY(d_lists.reserve(2 * kListMax * (size_t)N));
    LFR_TRY(d_slot.reserve(4 * (size_t)N));
    LFR_TRY(d_pool.reserve(8 * slots * U.W));
    LFR_TRY(d_pool_next.reserve(4));
    LFR_CUDA(cudaMemsetAsync(d_pool.p, 0, 8 * slots * U.W, s));
    LFR_CUDA(cudaMemsetAsync(d_pool_next.p, 0, 4, s));
    U.lists = d_lists.as<uint16_t>();
    U.slot = d_slot.as<int32_t>();
    U.pool = d_pool.as<unsigned long long>();
    U.pool_next = d_pool_next.as<uint32_t>();
  }
  uf_init_kernel<<<blocks_for(N), 256, 0, s>>>(U, N);
  LFR_LAUNCHED();
  {
    uint32_t w_max = 1u << 18;
    if (const char* e = std::getenv("LFR_KRUSKAL_WINDOW")) w_max = (uint32_t)std::max(1l, std::atol(e));
    w_max = (uint32_t)std::min<uint64_t>(w_max, M);
    TmpBuf win[2], wr1, wr2, wst, keep, nsel;
    LFR_TRY(win[0].reserve(4 * (size_t)w_max));
    LFR_TRY(win[1].reserve(4 * (size_t)w_max));
    LFR_TRY(wr1.reserve(4 * (size_t)w_max));
    LFR_TRY(wr2.reserve(4 * (size_t)w_max));
    LFR_TRY(wst.reserve(w_max));
    LFR_TRY(keep.reserve(4 * (size_t)w_max));
    LFR_TRY(nsel.reserve(4));
    iota_kernel<<<blocks_for(w_max), 256, 0, s>>>(win[0].as<uint32_t>(), w_max);
    LFR_LAUNCHED();
    uint32_t n_win = w_max, next = w_max;
    int cur = 0;
    while (n_win) {
      uint32_t* w = win[cur].as<uint32_t>();
      uint32_t* w2 = win[1 - cur].as<uint32_t>();
      kr_reserve_kernel<<<blocks_for(n_win), 256, 0, s>>>(U, w, n_win, d_order.as<uint32_t>(), (uint32_t)M, d_nop.as<uint32_t>(),
                                                          wr1.as<uint32_t>(), wr2.as<uint32_t>(), wst.as<uint8_t>());
      kr_decide_kernel<<<blocks_for(n_win), 256, 0, s>>>(U, w, n_win, wr1.as<uint32_t>(), wr2.as<uint32_t>(), wst.as<uint8_t>());
      kr_release_kernel<<<blocks_for(n_win), 256, 0, s>>>(U, n_win, wr1.as<uint32_t>(), wr2.as<uint32_t>(), wst.as<uint8_t>(),
                                                          keep.as<uint32_t>());
      LFR_LAUNCHED();
      uint32_t *kp = keep.as<uint32_t>(), *ns_d = nsel.as<uint32_t>();
      const int nw = (int)n_win;
      LFR_TRY(cub_run(tmp, [&](void* t, size_t& nb) { return cub::DeviceSelect::Flagged(t, nb, w, kp, w2, ns_d, nw, s); }));
      uint32_t ns = 0;
      LFR_TRY(fetch(&ns, ns_d, 1, s));
      const uint32_t add = (uint32_t)std::min<uint64_t>(w_max - ns, M - next);
      if (add) {
        kr_refill_kernel<<<blocks_for(add), 256, 0, s>>>(w2, ns, add, next);
        LFR_LAUNCHED();
      }
      next += add;
      n_win = ns + add;
      cur = 1 - cur;
    }
  }
  // ---- H3: track ids (roots in node order) and roots ---------------------------------------------------
  TmpBuf d_flag, d_tid, d_nit, d_score, d_best, d_bestnode, d_red;
  uint32_t T = 0;
  LFR_TRY(d_flag.reserve(4 * ((size_t)N + 1)));
  LFR_TRY(d_tid.reserve(4 * ((size_t)N + 1)));
  root_flags_kernel<<<blocks_for(N), 256, 0, s>>>(d_parent.as<int32_t>(), N, d_flag.as<uint32_t>());
  LFR_LAUNCHED();
  LFR_CUDA(cudaMemsetAsync(d_flag.as<uint32_t>() + N, 0, 4, s));
  {
    uint32_t *f = d_flag.as<uint32_t>(), *tid = d_tid.as<uint32_t>();
    LFR_TRY(cub_run(tmp, [&](void* t, size_t& nb) { return cub::DeviceScan::ExclusiveSum(t, nb, f, tid, (int)N + 1, s); }));
    LFR_TRY(fetch(&T, tid + N, 1, s));
  }
  LFR_TRY(d_track.reserve(4 * (size_t)N));
  LFR_TRY(d_nit.reserve(4 * (size_t)T));
  LFR_CUDA(cudaMemsetAsync(d_nit.p, 0, 4 * (size_t)T, s));
  track_ids_kernel<<<blocks_for(N), 256, 0, s>>>(d_parent.as<int32_t>(), d_tid.as<uint32_t>(), N, d_track.as<uint32_t>(),
                                                 d_nit.as<uint32_t>());
  LFR_LAUNCHED();
  LFR_TRY(d_red.reserve(8));
  {
    uint32_t *nit = d_nit.as<uint32_t>(), *out = d_red.as<uint32_t>();
    LFR_TRY(cub_run(tmp, [&](void* t, size_t& nb) { return cub::DeviceReduce::Reduce(t, nb, nit, out, (int)T, MaxOp(), 0u, s); }));
    LFR_TRY(fetch(&S->max_track_size, out, 1, s));
  }
  LFR_TRY(d_score.reserve(8 * (size_t)N));
  LFR_TRY(d_best.reserve(8 * (size_t)T));
  LFR_TRY(d_bestnode.reserve(4 * (size_t)T));
  LFR_TRY(d_isroot.reserve(N));
  LFR_CUDA(cudaMemsetAsync(d_best.p, 0, 8 * (size_t)T, s));
  LFR_CUDA(cudaMemsetAsync(d_bestnode.p, 0, 4 * (size_t)T, s));
  LFR_CUDA(cudaMemsetAsync(d_isroot.p, 0, N, s));
  root_score_kernel<<<blocks_for(N), 256, 0, s>>>(d_rowptr.as<uint32_t>(), d_cdst.as<uint32_t>(), d_csim.as<float>(),
                                                  d_track.as<uint32_t>(), N, d_score.as<double>(), d_best.as<unsigned long long>());
  root_pick_kernel<<<blocks_for(N), 256, 0, s>>>(d_score.as<double>(), d_best.as<unsigned long long>(), d_track.as<uint32_t>(), N,
                                                 d_bestnode.as<uint32_t>());
  root_mark_kernel<<<blocks_for(T), 256, 0, s>>>(d_bestnode.as<uint32_t>(), T, d_isroot.as<uint8_t>());
  LFR_LAUNCHED();
  LFR_CUDA(cudaStreamSynchronize(s));
  S->tracks_ms = ms_since(t_tracks);
  const auto t_cut = Clock::now();
  // ---- H4: meta-graph: inter-track edges in CSR order, stable-sorted by (source, destination) track ----
  d_parent.release();
  d_size.release();
  d_res.release();
  d_mask.release();
  d_lists.release();
  d_pool.release();
  TmpBuf d_mkey, d_inter, d_ikey, d_ikey2, d_isim, d_isim2, d_nint, d_seg, d_nseg, d_ma, d_mb, d_wsum;
  uint32_t n_inter = 0, n_meta = 0;
  LFR_TRY(d_mkey.reserve(8 * E));
  LFR_TRY(d_inter.reserve(4 * E));
  meta_keys_kernel<<<blocks_for(E), 256, 0, s>>>(d_ssrc.as<uint32_t>(), d_cdst.as<uint32_t>(), d_track.as<uint32_t>(), E, T,
                                                 d_mkey.as<unsigned long long>(), d_inter.as<uint32_t>());
  LFR_LAUNCHED();
  LFR_TRY(d_ikey.reserve(8 * E));
  LFR_TRY(d_isim.reserve(4 * E));
  LFR_TRY(d_nint.reserve(4));
  {
    unsigned long long *mk = d_mkey.as<unsigned long long>(), *ik = d_ikey.as<unsigned long long>();
    uint32_t *fl = d_inter.as<uint32_t>(), *cnt = d_nint.as<uint32_t>();
    float *cs = d_csim.as<float>(), *is = d_isim.as<float>();
    LFR_TRY(cub_run(tmp, [&](void* t, size_t& nb) { return cub::DeviceSelect::Flagged(t, nb, mk, fl, ik, cnt, (int)E, s); }));
    LFR_TRY(cub_run(tmp, [&](void* t, size_t& nb) { return cub::DeviceSelect::Flagged(t, nb, cs, fl, is, cnt, (int)E, s); }));
    LFR_TRY(fetch(&n_inter, cnt, 1, s));
  }
  if (n_inter) {
    LFR_TRY(d_ikey2.reserve(8 * (size_t)n_inter));
    LFR_TRY(d_isim2.reserve(4 * (size_t)n_inter));
    LFR_TRY(d_seg.reserve(4 * (size_t)n_inter));
    LFR_TRY(d_nseg.reserve(4));
    unsigned long long *ik = d_ikey.as<unsigned long long>(), *ik2 = d_ikey2.as<unsigned long long>();
    float *is = d_isim.as<float>(), *is2 = d_isim2.as<float>();
    const int end_bit = bits_for((uint64_t)T * T - 1);
    LFR_TRY(cub_run(tmp, [&](void* t, size_t& nb) {
      return cub::DeviceRadixSort::SortPairs(t, nb, ik, ik2, is, is2, (int)n_inter, 0, end_bit, s);
    }));
    uint32_t* head = d_inter.as<uint32_t>();  // reused
    seg_heads_kernel<<<blocks_for(n_inter), 256, 0, s>>>(ik2, n_inter, head);
    LFR_LAUNCHED();
    uint32_t *seg = d_seg.as<uint32_t>(), *cnt = d_nseg.as<uint32_t>();
    uint32_t* idx = d_pos.as<uint32_t>();  // 0, 1, ... (n_inter <= E)
    iota_kernel<<<blocks_for(n_inter), 256, 0, s>>>(idx, n_inter);
    LFR_LAUNCHED();
    LFR_TRY(cub_run(tmp, [&](void* t, size_t& nb) { return cub::DeviceSelect::Flagged(t, nb, idx, head, seg, cnt, (int)n_inter, s); }));
    LFR_TRY(fetch(&n_meta, cnt, 1, s));
    LFR_TRY(d_ma.reserve(4 * (size_t)n_meta));
    LFR_TRY(d_mb.reserve(4 * (size_t)n_meta));
    LFR_TRY(d_wsum.reserve(8 * (size_t)n_meta));
    meta_sum_kernel<<<blocks_for(n_meta), 256, 0, s>>>(ik2, is2, seg, n_meta, n_inter, T, d_ma.as<uint32_t>(), d_mb.as<uint32_t>(),
                                                       d_wsum.as<double>());
    LFR_LAUNCHED();
  }
  // components of the meta-graph, the oversized ones cut on the host, the final components
  TmpBuf d_cc, d_ccn, d_big, d_gc, d_fcc;
  uint32_t n_cc = 0, n_final = 0;
  LFR_TRY(d_cc.reserve(4 * (size_t)T));
  LFR_TRY(components_on_device(T, d_ma.as<uint32_t>(), d_mb.as<uint32_t>(), n_meta, nullptr, d_cc.as<uint32_t>(), &n_cc, tmp, s));
  S->n_meta_components = n_cc;
  LFR_TRY(d_ccn.reserve(8 * (size_t)n_cc));
  LFR_TRY(d_big.reserve(4 * (size_t)n_cc));
  LFR_CUDA(cudaMemsetAsync(d_ccn.p, 0, 8 * (size_t)n_cc, s));
  cc_weight_kernel<<<blocks_for(T), 256, 0, s>>>(d_cc.as<uint32_t>(), d_nit.as<uint32_t>(), T, d_ccn.as<unsigned long long>());
  // sub-scenes: the cap of every meta-component and of each of its tracks
  TmpBuf d_icap, d_cccap, d_tcap;
  if (group) {
    LFR_TRY(upload(&d_icap, image_cap.data(), n_images, s));
    LFR_TRY(d_cccap.reserve(4 * (size_t)n_cc));
    LFR_TRY(d_tcap.reserve(4 * (size_t)T));
    cc_cap_kernel<<<blocks_for(N), 256, 0, s>>>(d_nimg.as<uint32_t>(), d_track.as<uint32_t>(), d_cc.as<uint32_t>(),
                                                 d_icap.as<uint32_t>(), N, d_cccap.as<uint32_t>());
    gather_kernel<<<blocks_for(T), 256, 0, s>>>(d_cc.as<uint32_t>(), d_cccap.as<uint32_t>(), T, d_tcap.as<uint32_t>());
    LFR_LAUNCHED();
  }
  oversized_kernel<<<blocks_for(n_cc), 256, 0, s>>>(d_ccn.as<unsigned long long>(), n_cc, S->n_images_seen,
                                                    group ? d_cccap.as<uint32_t>() : nullptr, d_big.as<uint32_t>());
  LFR_LAUNCHED();
  {
    uint32_t *big = d_big.as<uint32_t>(), *out = d_red.as<uint32_t>();
    LFR_TRY(cub_run(tmp, [&](void* t, size_t& nb) { return cub::DeviceReduce::Sum(t, nb, big, out, (int)n_cc, s); }));
    LFR_TRY(fetch(&S->n_oversized_meta_components, out, 1, s));
  }
  LFR_TRY(d_gc.reserve(4 * (size_t)T));
  LFR_CUDA(cudaMemcpyAsync(d_gc.p, d_cc.p, 4 * (size_t)T, cudaMemcpyDeviceToDevice, s));
  if (S->n_oversized_meta_components) {
    // the undirected edges of the oversized components, in meta-edge order, to the cut
    TmpBuf d_cflag, d_cidx, d_ncut, d_recs, d_gidx, d_gval;
    uint32_t n_cut = 0;
    LFR_TRY(d_cflag.reserve(4 * (size_t)n_meta));
    LFR_TRY(d_cidx.reserve(4 * (size_t)n_meta));
    LFR_TRY(d_ncut.reserve(4));
    cut_edges_flag_kernel<<<blocks_for(n_meta), 256, 0, s>>>(d_ma.as<uint32_t>(), d_mb.as<uint32_t>(), d_cc.as<uint32_t>(),
                                                            d_big.as<uint32_t>(), n_meta, d_cflag.as<uint32_t>());
    LFR_LAUNCHED();
    uint32_t *fl = d_cflag.as<uint32_t>(), *ci = d_cidx.as<uint32_t>(), *cnt = d_ncut.as<uint32_t>();
    uint32_t* idx = d_pos.as<uint32_t>();  // 0, 1, ... (n_meta <= E)
    iota_kernel<<<blocks_for(n_meta), 256, 0, s>>>(idx, n_meta);
    LFR_LAUNCHED();
    LFR_TRY(cub_run(tmp, [&](void* t, size_t& nb) { return cub::DeviceSelect::Flagged(t, nb, idx, fl, ci, cnt, (int)n_meta, s); }));
    LFR_TRY(fetch(&n_cut, cnt, 1, s));
    if (device_cut) {
      // lfr_cut.cuh: the roots are the oversized components, the labels go straight into d_gc
      CutLists E[2];
      TmpBuf d_rkey, d_ridx;
      LFR_TRY(E[0].reserve(n_cut));
      LFR_TRY(E[1].reserve(n_cut));
      LFR_TRY(d_rkey.reserve(4 * (size_t)n_cut));
      LFR_TRY(d_ridx.reserve(4 * (size_t)n_cut));
      lfr::cut::root_edges_kernel<<<blocks_for(n_cut), 256, 0, s>>>(ci, n_cut, d_ma.as<uint32_t>(), d_mb.as<uint32_t>(), d_wsum.as<double>(),
                                                                    d_cc.as<uint32_t>(), E[1].a.as<uint32_t>(), E[1].b.as<uint32_t>(),
                                                                    E[1].w.as<long long>(), d_rkey.as<uint32_t>(), d_ridx.as<uint32_t>());
      LFR_LAUNCHED();
      uint32_t n_roots = 0;
      LFR_TRY(group_cut_edges(d_rkey.as<uint32_t>(), d_ridx.as<uint32_t>(), n_cut, bits_for(std::max<uint32_t>(n_cc, 2) - 1), E[1], E[0],
                              &n_roots, tmp, s));
      LFR_TRY(recursive_cut_on_device(T, E, n_cut, n_roots, d_nit.as<uint32_t>(), S->n_images_seen, n_cc, d_gc.as<uint32_t>(),
                                      &S->n_cut_groups, tmp, s, group ? d_tcap.as<uint32_t>() : nullptr));
    } else {
      LFR_TRY(d_recs.reserve(sizeof(CutRec) * std::max<size_t>(n_cut, 1)));
      if (n_cut) {
        cut_edges_gather_kernel<<<blocks_for(n_cut), 256, 0, s>>>(ci, n_cut, d_ma.as<uint32_t>(), d_mb.as<uint32_t>(),
                                                                  d_wsum.as<double>(), d_cc.as<uint32_t>(), d_recs.as<CutRec>());
        LFR_LAUNCHED();
      }
      std::vector<CutRec> recs(n_cut);
      std::vector<uint32_t> node_weight(T);
      LFR_TRY(fetch(recs.data(), d_recs.p, n_cut, s));
      LFR_TRY(fetch(node_weight.data(), d_nit.p, T, s));
      // one edge list per oversized component, components ascending (lfr_host.cc's per_cc)
      std::vector<uint32_t> comps;
      for (const CutRec& r : recs) comps.push_back(r.comp);
      std::sort(comps.begin(), comps.end());
      comps.erase(std::unique(comps.begin(), comps.end()), comps.end());
      std::vector<std::vector<lfr::CutEdge>> per_cc(comps.size());
      for (const CutRec& r : recs) {
        const size_t sl = (size_t)(std::lower_bound(comps.begin(), comps.end(), r.comp) - comps.begin());
        per_cc[sl].push_back(lfr::CutEdge{r.a, r.b, lfr::cut_weight(r.wsum)});
      }
      std::vector<uint32_t> track_cap(group ? T : 0);
      if (group) LFR_TRY(fetch(track_cap.data(), d_tcap.p, T, s));
      std::vector<std::vector<uint32_t>> groups;
      lfr::recursive_cut_all(std::move(per_cc), node_weight, S->n_images_seen, &groups, group ? track_cap.data() : nullptr);
      std::vector<uint32_t> gidx, gval;
      for (size_t g = 0; g < groups.size(); ++g)
        for (uint32_t t : groups[g]) {
          gidx.push_back(t);
          gval.push_back(n_cc + (uint32_t)g);
        }
      S->n_cut_groups = (uint32_t)groups.size();
      if (!gidx.empty()) {
        LFR_TRY(upload(&d_gidx, gidx.data(), gidx.size(), s));
        LFR_TRY(upload(&d_gval, gval.data(), gval.size(), s));
        scatter_kernel<<<blocks_for(gidx.size()), 256, 0, s>>>(d_gidx.as<uint32_t>(), d_gval.as<uint32_t>(), (uint32_t)gidx.size(),
                                                               d_gc.as<uint32_t>());
        LFR_LAUNCHED();
      }
      LFR_CUDA(cudaStreamSynchronize(s));  // the uploads above read host vectors that end with this scope
    }
  }
  LFR_TRY(d_fcc.reserve(4 * (size_t)T));
  LFR_TRY(components_on_device(T, d_ma.as<uint32_t>(), d_mb.as<uint32_t>(), n_meta, d_gc.as<uint32_t>(), d_fcc.as<uint32_t>(),
                               &n_final, tmp, s));
  LFR_TRY(d_comp.reserve(4 * (size_t)N));
  gather_kernel<<<blocks_for(N), 256, 0, s>>>(d_track.as<uint32_t>(), d_fcc.as<uint32_t>(), N, d_comp.as<uint32_t>());
  LFR_LAUNCHED();
  LFR_CUDA(cudaStreamSynchronize(s));
  S->graph_cut_ms = ms_since(t_cut);
  const auto t_disp = Clock::now();
  // ---- H5: dispatch list: slots by (size desc, id desc), nodes ascending inside a slot ----------------
  const uint32_t C = n_final;
  TmpBuf d_csize, d_ckey, d_ckey2, d_corder, d_slotof, d_ssize, d_nslot, d_nslot2, d_iota;
  LFR_TRY(d_csize.reserve(4 * (size_t)C));
  LFR_TRY(d_ckey.reserve(8 * (size_t)C));
  LFR_TRY(d_ckey2.reserve(8 * (size_t)C));
  LFR_TRY(d_corder.reserve(4 * (size_t)C));
  LFR_TRY(d_slotof.reserve(4 * (size_t)C));
  LFR_TRY(d_ssize.reserve(4 * ((size_t)C + 1)));
  LFR_TRY(d_cptr.reserve(4 * ((size_t)C + 1)));
  LFR_CUDA(cudaMemsetAsync(d_csize.p, 0, 4 * (size_t)C, s));
  LFR_CUDA(cudaMemsetAsync(d_ssize.p, 0, 4 * ((size_t)C + 1), s));
  comp_size_kernel<<<blocks_for(N), 256, 0, s>>>(d_comp.as<uint32_t>(), N, d_csize.as<uint32_t>());
  comp_keys_kernel<<<blocks_for(C), 256, 0, s>>>(d_csize.as<uint32_t>(), C, d_ckey.as<unsigned long long>());
  LFR_LAUNCHED();
  {
    unsigned long long *k1 = d_ckey.as<unsigned long long>(), *k2 = d_ckey2.as<unsigned long long>();
    const int end_bit = 32 + bits_for(N);
    LFR_TRY(cub_run(tmp, [&](void* t, size_t& nb) { return cub::DeviceRadixSort::SortKeysDescending(t, nb, k1, k2, (int)C, 0, end_bit, s); }));
    comp_slots_kernel<<<blocks_for(C), 256, 0, s>>>(k2, C, d_corder.as<uint32_t>(), d_slotof.as<uint32_t>(), d_ssize.as<uint32_t>());
    LFR_LAUNCHED();
    uint32_t *ss = d_ssize.as<uint32_t>(), *cp = d_cptr.as<uint32_t>();
    LFR_TRY(cub_run(tmp, [&](void* t, size_t& nb) { return cub::DeviceScan::ExclusiveSum(t, nb, ss, cp, (int)C + 1, s); }));
  }
  LFR_TRY(d_nslot.reserve(4 * (size_t)N));
  LFR_TRY(d_nslot2.reserve(4 * (size_t)N));
  LFR_TRY(d_cnodes.reserve(4 * (size_t)N));
  LFR_TRY(d_iota.reserve(4 * (size_t)N));
  node_slot_kernel<<<blocks_for(N), 256, 0, s>>>(d_comp.as<uint32_t>(), d_slotof.as<uint32_t>(), N, d_nslot.as<uint32_t>());
  iota_kernel<<<blocks_for(N), 256, 0, s>>>(d_iota.as<uint32_t>(), N);
  LFR_LAUNCHED();
  {
    uint32_t *k1 = d_nslot.as<uint32_t>(), *k2 = d_nslot2.as<uint32_t>(), *v1 = d_iota.as<uint32_t>(), *v2 = d_cnodes.as<uint32_t>();
    const int end_bit = bits_for(C);
    LFR_TRY(cub_run(tmp, [&](void* t, size_t& nb) { return cub::DeviceRadixSort::SortPairs(t, nb, k1, k2, v1, v2, (int)N, 0, end_bit, s); }));
  }
  // the per-node arrays to the host: the schedule builder and lfr_plan_export_graph() read them
  G->row_ptr.resize((size_t)N + 1);
  G->track.resize(N);
  G->comp.resize(N);
  G->is_root.resize(N);
  G->comp_ptr.resize((size_t)C + 1);
  G->comp_nodes.resize(N);
  G->comp_order.resize(C);
  G->node_image.resize(N);
  G->node_feat.resize(N);
  LFR_CUDA(cudaMemcpyAsync(G->row_ptr.data(), d_rowptr.p, 4 * ((size_t)N + 1), cudaMemcpyDeviceToHost, s));
  LFR_CUDA(cudaMemcpyAsync(G->track.data(), d_track.p, 4 * (size_t)N, cudaMemcpyDeviceToHost, s));
  LFR_CUDA(cudaMemcpyAsync(G->comp.data(), d_comp.p, 4 * (size_t)N, cudaMemcpyDeviceToHost, s));
  LFR_CUDA(cudaMemcpyAsync(G->is_root.data(), d_isroot.p, N, cudaMemcpyDeviceToHost, s));
  LFR_CUDA(cudaMemcpyAsync(G->comp_ptr.data(), d_cptr.p, 4 * ((size_t)C + 1), cudaMemcpyDeviceToHost, s));
  LFR_CUDA(cudaMemcpyAsync(G->comp_nodes.data(), d_cnodes.p, 4 * (size_t)N, cudaMemcpyDeviceToHost, s));
  LFR_CUDA(cudaMemcpyAsync(G->comp_order.data(), d_corder.p, 4 * (size_t)C, cudaMemcpyDeviceToHost, s));
  LFR_CUDA(cudaMemcpyAsync(G->node_image.data(), d_nimg.p, 4 * (size_t)N, cudaMemcpyDeviceToHost, s));
  LFR_CUDA(cudaMemcpyAsync(G->node_feat.data(), d_nfeat.p, 4 * (size_t)N, cudaMemcpyDeviceToHost, s));
  LFR_CUDA(cudaStreamSynchronize(s));
  S->dispatch_ms = ms_since(t_disp);
  S->n_nodes = N;
  S->n_edges = E;
  S->n_tracks = T;
  S->n_components = C;
  S->max_component_size = C ? G->comp_ptr[1] - G->comp_ptr[0] : 0;
  pl->graph = std::move(G);
  return LFR_OK;
}

// lfr_plan_create_from_matches(): the decoded match arrays of `in` go up as they are
int upload_matches(const lfr_host_input* in, MatchArrays& d, cudaStream_t s) {
  const size_t M = in->n_matches;
  LFR_TRY(upload(&d.feat1, in->feat1, M, s));
  LFR_TRY(upload(&d.feat2, in->feat2, M, s));
  LFR_TRY(upload(&d.sim, in->sim, M, s));
  LFR_TRY(upload(&d.disp1, in->disp1, 18 * M, s));
  LFR_TRY(upload(&d.disp2, in->disp2, 18 * M, s));
  return LFR_OK;
}

// Host -> device copies of caller memory that may be pageable (a mapped file): through two page-locked
// chunks, so that the host copy into one overlaps the DMA out of the other.
struct Stager {
  static constexpr size_t kChunk = 8u << 20;
  uint8_t* h[2] = {};
  cudaEvent_t ev[2] = {};
  size_t chunk = 0;
  int k = 0;
  int init(size_t largest) {
    chunk = std::max<size_t>(std::min(kChunk, largest), 1);
    for (int i = 0; i < 2; ++i) {
      LFR_CUDA(cudaHostAlloc((void**)&h[i], chunk, cudaHostAllocDefault));
      LFR_CUDA(cudaEventCreateWithFlags(&ev[i], cudaEventDisableTiming));
    }
    return LFR_OK;
  }
  int put(void* dst, const void* src, size_t bytes, cudaStream_t s) {
    for (size_t o = 0; o < bytes; o += chunk) {
      const size_t b = std::min(chunk, bytes - o);
      LFR_CUDA(cudaEventSynchronize(ev[k]));  // this chunk's previous DMA has finished
      std::memcpy(h[k], static_cast<const uint8_t*>(src) + o, b);
      LFR_CUDA(cudaMemcpyAsync(static_cast<uint8_t*>(dst) + o, h[k], b, cudaMemcpyHostToDevice, s));
      LFR_CUDA(cudaEventRecord(ev[k], s));
      k ^= 1;
    }
    return LFR_OK;
  }
  ~Stager() {
    for (int i = 0; i < 2; ++i) {
      if (ev[i]) {
        cudaEventSynchronize(ev[i]);
        cudaEventDestroy(ev[i]);
      }
      if (h[i]) cudaFreeHost(h[i]);
    }
  }
};

// {staging + copy, decode kernels} in ms of the calling thread's last lfr_plan_create_from_wire()
thread_local double g_wire_ms[2] = {};

// lfr_plan_create_from_wire(): every part's bytes and match offsets go up through the stager and every
// Match is decoded on the device into `d` at its global index (parts in order).  LFR_EINVAL when a match
// is malformed, before the graph stage sees anything.
int decode_wire_on_device(const lfr_host_input* in, const lfr_wire_part* parts, uint32_t n_parts, MatchArrays& d,
                          cudaStream_t s) {
  g_wire_ms[0] = g_wire_ms[1] = 0;
  const size_t M = in->n_matches;
  uint64_t total = 0;
  size_t max_len = 0, max_n = 0;
  for (uint32_t i = 0; i < n_parts; ++i) {
    const lfr_wire_part& pt = parts[i];
    if ((!pt.buf && pt.len) || (!pt.match_off && pt.n_matches)) return fail(LFR_EINVAL, "NULL part buffer or match offsets");
    total += pt.n_matches;
    if (pt.n_matches) {
      max_len = std::max<size_t>(max_len, pt.len);
      max_n = std::max<size_t>(max_n, pt.n_matches);
    }
  }
  if (total != M) return fail(LFR_EINVAL, "the parts' match counts do not add up to n_matches");
  LFR_TRY(d.feat1.reserve(4 * std::max<size_t>(M, 1)));
  LFR_TRY(d.feat2.reserve(4 * std::max<size_t>(M, 1)));
  LFR_TRY(d.sim.reserve(4 * std::max<size_t>(M, 1)));
  LFR_TRY(d.disp1.reserve(72 * std::max<size_t>(M, 1)));
  LFR_TRY(d.disp2.reserve(72 * std::max<size_t>(M, 1)));
  if (!M) return LFR_OK;
  const auto t0 = Clock::now();
  LFR_CUDA(cudaMemsetAsync(d.disp1.p, 0, 72 * M, s));
  LFR_CUDA(cudaMemsetAsync(d.disp2.p, 0, 72 * M, s));
  TmpBuf d_bytes, d_moff, d_err;
  LFR_TRY(d_bytes.reserve(std::max<size_t>(max_len, 1)));
  LFR_TRY(d_moff.reserve(8 * max_n));
  LFR_TRY(d_err.reserve(4));
  LFR_CUDA(cudaMemsetAsync(d_err.p, 0, 4, s));
  Stager st;
  LFR_TRY(st.init(std::max<size_t>(max_len, 8 * max_n)));
  std::vector<cudaEvent_t> ev;
  struct EventsFree {
    std::vector<cudaEvent_t>& v;
    ~EventsFree() { for (cudaEvent_t e : v) cudaEventDestroy(e); }
  } ev_free{ev};
  uint64_t m0 = 0;
  for (uint32_t i = 0; i < n_parts; ++i) {
    const lfr_wire_part& pt = parts[i];
    if (!pt.n_matches) continue;
    LFR_TRY(st.put(d_bytes.p, pt.buf, pt.len, s));
    LFR_TRY(st.put(d_moff.p, pt.match_off, 8 * pt.n_matches, s));
    cudaEvent_t e[2];
    for (cudaEvent_t& x : e) {
      LFR_CUDA(cudaEventCreate(&x));
      ev.push_back(x);
    }
    LFR_CUDA(cudaEventRecord(e[0], s));
    lfr::wire::decode_matches_kernel<<<blocks_for(pt.n_matches), 256, 0, s>>>(
        d_bytes.as<uint8_t>(), pt.len, d_moff.as<uint64_t>(), pt.n_matches, m0, d.feat1.as<uint32_t>(),
        d.feat2.as<uint32_t>(), d.sim.as<float>(), d.disp1.as<float>(), d.disp2.as<float>(), d_err.as<int>());
    LFR_LAUNCHED();
    LFR_CUDA(cudaEventRecord(e[1], s));
    m0 += pt.n_matches;
  }
  int err = 0;
  LFR_TRY(fetch(&err, d_err.p, 1, s));
  for (size_t j = 0; j < ev.size(); j += 2) {
    float ms = 0.f;
    LFR_CUDA(cudaEventElapsedTime(&ms, ev[j], ev[j + 1]));
    g_wire_ms[1] += ms;
  }
  g_wire_ms[0] = ms_since(t0) - g_wire_ms[1];
  if (err) return fail(LFR_EINVAL, kMalformedMatch);
  return LFR_OK;
}

// lfr_plan_create_from_wire_listed(): the batch's match arrays `d` (M matches) from the file's, `src`, decoded
// once in file order.  A scan of the entries' match counts gives each entry's first match; one block per
// entry then copies its source pair's matches there, bit for bit.
int expand_listed_on_device(const uint64_t* src_pair_ptr, uint64_t n_src, const uint64_t* pair_src, uint64_t n,
                            uint64_t M, const MatchArrays& src, MatchArrays& d, cudaStream_t s) {
  LFR_TRY(d.feat1.reserve(4 * std::max<size_t>(M, 1)));
  LFR_TRY(d.feat2.reserve(4 * std::max<size_t>(M, 1)));
  LFR_TRY(d.sim.reserve(4 * std::max<size_t>(M, 1)));
  LFR_TRY(d.disp1.reserve(72 * std::max<size_t>(M, 1)));
  LFR_TRY(d.disp2.reserve(72 * std::max<size_t>(M, 1)));
  if (!M) return LFR_OK;
  TmpBuf d_sptr, d_psrc, d_cnt, d_dst, tmp;
  LFR_TRY(upload(&d_sptr, src_pair_ptr, n_src + 1, s));
  LFR_TRY(upload(&d_psrc, pair_src, n, s));
  LFR_TRY(d_cnt.reserve(8 * (n + 1)));
  LFR_TRY(d_dst.reserve(8 * (n + 1)));
  uint64_t* cnt = d_cnt.as<uint64_t>();
  uint64_t* dst = d_dst.as<uint64_t>();
  lfr::wire::listed_counts_kernel<<<blocks_for(n + 1), 256, 0, s>>>(d_sptr.as<uint64_t>(), d_psrc.as<uint64_t>(), n, cnt);
  LFR_LAUNCHED();
  LFR_TRY(cub_run(tmp, [&](void* t, size_t& nb) { return cub::DeviceScan::ExclusiveSum(t, nb, cnt, dst, (int)n + 1, s); }));
  const unsigned grid = (unsigned)std::min<uint64_t>(n, 1u << 30);
  lfr::wire::listed_gather_kernel<<<grid, 256, 0, s>>>(
      d_sptr.as<uint64_t>(), d_psrc.as<uint64_t>(), dst, n, src.feat1.as<uint32_t>(), src.feat2.as<uint32_t>(),
      src.sim.as<uint32_t>(), src.disp1.as<uint2>(), src.disp2.as<uint2>(), d.feat1.as<uint32_t>(),
      d.feat2.as<uint32_t>(), d.sim.as<uint32_t>(), d.disp1.as<uint2>(), d.disp2.as<uint2>());
  LFR_LAUNCHED();
  LFR_CUDA(cudaStreamSynchronize(s));  // before the scratch buffers and `src` are freed
  return LFR_OK;
}

// The two entry points from matches: the stage on the device-resident `d`, then the plan.
int create_plan_from_graph(const lfr_host_input* in, MatchArrays& d, const lfr_options& o, const double* initial_positions,
                           lfr_plan* pl, lfr_host_sizes* S) {
  LFR_TRY(build_graph_on_device(in, d, pl, S, (o.debug_flags & LFR_DBG_DEVICE_CUT) != 0, 0));
  const lfr_plan::GraphArrays& G = *pl->graph;
  lfr_problem p;
  p.n_nodes = S->n_nodes;
  p.n_components = S->n_components;
  p.n_edges = S->n_edges;
  p.row_ptr = G.row_ptr.data();
  p.edges = nullptr;  // already in pl->edges
  p.track = G.track.data();
  p.comp = G.comp.data();
  p.is_root = G.is_root.data();
  p.comp_ptr = G.comp_ptr.data();
  p.comp_nodes = G.comp_nodes.data();
  LFR_TRY(fill_plan(pl, &p, o, initial_positions, 0, false, nullptr, nullptr, /*graph_resident=*/true));
  // the working positions hold the start point from creation on, so lfr_plan_download() and
  // lfr_plan_encode_solution() see it before the first solve; that solve then skips its reset copy
  if (pl->N) {
    LFR_CUDA(cudaMemcpyAsync(pl->pos.p, pl->pos_init.p, sizeof(double) * 2 * (size_t)pl->N, cudaMemcpyDeviceToDevice, 0));
    pl->pos_is_staged = true;
  }
  pl->n_images = in->n_images;
  LFR_CUDA(cudaStreamSynchronize(0));
  return LFR_OK;
}

int set_kernel_attrs() {
  static bool done_for_device[16] = {};  // per device, guarded by that device's workspace mutex / idempotent otherwise
  int dev = 0;
  LFR_CUDA(cudaGetDevice(&dev));
  if (dev >= 0 && dev < 16 && done_for_device[dev]) return LFR_OK;
  for (const KernelInfo& k : kKernels)
    LFR_CUDA(cudaFuncSetAttribute(k.fn, cudaFuncAttributeMaxDynamicSharedMemorySize, k.smem_max));
  if (dev >= 0 && dev < 16) done_for_device[dev] = true;
  return LFR_OK;
}

int launch_solve(lfr_plan* pl, cudaStream_t s) {
  LFR_TRY(set_kernel_attrs());
  if (pl->N && !pl->pos_is_staged)
    LFR_CUDA(cudaMemcpyAsync(pl->pos.p, pl->pos_init.p, sizeof(double) * 2 * (size_t)pl->N,
                             cudaMemcpyDeviceToDevice, s));
  pl->pos_is_staged = false;  // a second launch on the same plan needs the reset again
  if (pl->profile && pl->C) {
    // the records are accumulated into (atomicAdd of cycles and of the tier word) and a component without
    // free nodes writes none: each solve starts from zero, or the last solve's records would be mixed with
    // every earlier one (a refixed mask moves components between tiers and to EMPTY)
    LFR_CUDA(cudaMemsetAsync(pl->cycles.p, 0, sizeof(unsigned long long) * 8 * (size_t)pl->C, s));
    LFR_CUDA(cudaMemsetAsync(pl->times.p, 0, sizeof(unsigned long long) * 2 * (size_t)pl->C, s));
  }
  const lfr::DevProblem P_hbm = pl->dev();  // edges read from the HBM copy by global index
  lfr::DevProblem P_stage = P_hbm;          // edges pulled once into shared memory, possibly from the caller's pinned buffer
  if (pl->zc_edges) {
    P_stage.edges = pl->zc_edges;
    P_stage.pull_window = zero_copy_pull_window();
  }
  const lfr::CtaArrays A = pl->cta_arrays();
  // The CTA tier's launches (its components are the longest) on side streams forked from the caller's,
  // the first other launch on the caller's stream, the rest on side streams; one launch alone runs on
  // the caller's stream.
  const bool fork = pl->launches.size() > 1;
  if (fork) LFR_CUDA(cudaEventRecord(pl->ev_fork, s));
  int side = 0, n_queue = 0;
  bool caller_busy = false;
  for (const Launch& L : pl->launches) {
    const KernelInfo& I = info(L.kernel);
    cudaStream_t bs = s;
    if (fork && (is_cta(L.kernel) || caller_busy)) {
      bs = pl->streams[side++ % pl->n_streams];
      LFR_CUDA(cudaStreamWaitEvent(bs, pl->ev_fork, 0));
    }
    caller_busy = caller_busy || !is_cta(L.kernel);
    // with zero-copy edges, the HBM copy and the CTA tier's preparation on the copy stream (fill_plan)
    if (pl->zc_edges && (I.edges == Edges::kGlobal ? pl->edges_in_hbm : I.edges == Edges::kPrepared && pl->cta_from_hbm))
      LFR_CUDA(cudaStreamWaitEvent(bs, pl->ev_edges, 0));
    const lfr::DevProblem& P = I.edges == Edges::kStaged ? P_stage : P_hbm;
    const unsigned grid = (L.n + L.warps - 1) / L.warps, block = I.threads * L.warps;
    const size_t smem = (size_t)L.bytes * L.warps;
    const lfr::WarpBucket wb{pl->lists.as<uint32_t>() + L.offset, L.n, L.emax, L.ncmax, L.n2max, L.bytes};
    const lfr::Warp2Queue q{wb.list, L.n, L.bytes, pl->queue_ctr.as<uint32_t>() + 2 * n_queue};
    const lfr::CtaComp* comps = is_cta(L.kernel) ? pl->L_comps.as<lfr::CtaComp>() + L.offset : nullptr;
    const unsigned smem_doubles = (unsigned)(smem / sizeof(double));
    switch (L.kernel) {
      case Kernel::kWarp2x4_8: lfr::solve_warp2_kernel<4, 8><<<grid, block, smem, bs>>>(P, pl->K, wb); break;
      case Kernel::kWarp2x4_16: lfr::solve_warp2_kernel<4, 16><<<grid, block, smem, bs>>>(P, pl->K, wb); break;
      case Kernel::kWarp2x1_32: lfr::solve_warp2_kernel<1, 32><<<grid, block, smem, bs>>>(P, pl->K, wb); break;
      case Kernel::kQueue:  // one CTA per SM
        lfr::solve_warp2_queue_kernel<<<pl->n_sms, block, smem, bs>>>(P, pl->K, q);
        ++n_queue;
        break;
      case Kernel::kTile64x32: lfr::solve_tile_kernel<64, 32><<<grid, block, smem, bs>>>(P, pl->K, wb); break;
      case Kernel::kTile64x48: lfr::solve_tile_kernel<64, 48><<<grid, block, smem, bs>>>(P, pl->K, wb); break;
      case Kernel::kTile64x64: lfr::solve_tile_kernel<64, 64><<<grid, block, smem, bs>>>(P, pl->K, wb); break;
      case Kernel::kTile128x80: lfr::solve_tile_kernel<128, 80><<<grid, block, smem, bs>>>(P, pl->K, wb); break;
      case Kernel::kWarp4: lfr::solve_warp_kernel<4><<<grid, block, smem, bs>>>(P, pl->K, wb); break;
      case Kernel::kWarp1: lfr::solve_warp_kernel<1><<<grid, block, smem, bs>>>(P, pl->K, wb); break;
      case Kernel::kCta2: lfr::solve_cta_kernel<256, 2><<<grid, block, smem, bs>>>(P, pl->K, A, comps, smem_doubles); break;
      case Kernel::kCta3: lfr::solve_cta_kernel<256, 3><<<grid, block, smem, bs>>>(P, pl->K, A, comps, smem_doubles); break;
      case Kernel::kCta4: lfr::solve_cta_kernel<256, 4><<<grid, block, smem, bs>>>(P, pl->K, A, comps, smem_doubles); break;
      case Kernel::kCount: break;  // (not a kernel)
    }
    LFR_CUDA(cudaGetLastError());
  }
  for (int k = 0; k < std::min(side, pl->n_streams); ++k) {  // join the side streams
    LFR_CUDA(cudaEventRecord(pl->ev_join[k], pl->streams[k]));
    LFR_CUDA(cudaStreamWaitEvent(s, pl->ev_join[k], 0));
  }
  return LFR_OK;
}

int download(lfr_plan* pl, cudaStream_t s, double* positions, lfr_stats* st) {
  const size_t nb = pl->stats_bytes();
  if (pl->h_stage_cap < nb) {
    if (pl->h_stage) cudaFreeHost(pl->h_stage);
    pl->h_stage = nullptr;
    pl->h_stage_cap = 0;
    LFR_CUDA(cudaMallocHost(&pl->h_stage, nb + nb / 4));
    pl->h_stage_cap = nb + nb / 4;
  }
  LFR_CUDA(cudaMemcpyAsync(pl->h_stage, pl->stats.p, nb, cudaMemcpyDeviceToHost, s));
  LFR_CUDA(cudaStreamSynchronize(s));
  const size_t Cp = pl->Cp;
  const double* h_cost0 = static_cast<const double*>(pl->h_stage);
  const double* h_cost1 = h_cost0 + Cp;
  const int32_t* h_iter = reinterpret_cast<const int32_t*>(h_cost1 + Cp);
  const int32_t* h_term = h_iter + Cp;
  const uint32_t* h_ls = reinterpret_cast<const uint32_t*>(h_term + Cp);
  const uint32_t* h_kept = h_ls + Cp;
  const int err = *reinterpret_cast<const int*>(h_kept + Cp);
  // the error flag is checked BEFORE anything is copied into the caller's position array (with
  // zero-copy write-back the components that did solve have already been written: on LFR_EINVAL
  // the array holds a mixture of start values and results)
  if (err)
    return fail(LFR_EINVAL, "edge with dst out of range, a self edge, or a component node list (comp_nodes) that "
                            "disagrees with comp (found while classifying edges on the device)");
  if (positions && pl->N && !pl->zc_positions) {
    LFR_CUDA(cudaMemcpyAsync(positions, pl->pos.p, sizeof(double) * 2 * (size_t)pl->N, cudaMemcpyDeviceToHost, s));
    LFR_CUDA(cudaStreamSynchronize(s));
  }
  if (st) {
    uint64_t ti = 0, tl = 0;
    for (uint32_t c = 0; c < pl->C; ++c) {
      ti += (uint64_t)h_iter[c];
      tl += h_ls[c];
    }
    if (pl->C) {
      if (st->iterations) std::memcpy(st->iterations, h_iter, sizeof(int32_t) * pl->C);
      if (st->termination) std::memcpy(st->termination, h_term, sizeof(int32_t) * pl->C);
      if (st->initial_cost) std::memcpy(st->initial_cost, h_cost0, sizeof(double) * pl->C);
      if (st->final_cost) std::memcpy(st->final_cost, h_cost1, sizeof(double) * pl->C);
    }
    st->total_iterations = ti;
    st->total_line_search_steps = tl;
    st->n_solved = pl->n_solved;
    st->n_kernel_launches = (uint32_t)pl->num_launches();
  }
  return LFR_OK;
}

// {kernels and the upload of names and facts, device-to-host copy of the bytes} in ms of the calling
// thread's last lfr_plan_encode_solution* call that wrote its output
thread_local double g_encode_ms[2] = {};

// Device arrays carved out of one buffer at 256-byte boundaries: `lay` takes every array in turn with
// take<T>(count); it runs once to size the buffer and once more to place the arrays in it.
struct Carve {
  uintptr_t base = 0;
  size_t at = 0;
  template <typename T>
  T* take(size_t count) {
    T* p = reinterpret_cast<T*>(base + at);
    at += (sizeof(T) * count + 255) & ~(size_t)255;
    return p;
  }
};

template <typename F>
int carve(DevBuf& buf, F&& lay) {
  Carve c;
  lay(c);
  LFR_TRY(buf.reserve(c.at));
  c = Carve{reinterpret_cast<uintptr_t>(buf.p), 0};
  lay(c);
  return LFR_OK;
}

// The checks of every call that reads the scene's image names, in this order: a plan made from matches,
// n_images, the caller's NULL arguments (`missing`: the message for the one found, or NULL), ascending
// name_off (and, with `group`, every image's group below G) and names.
int check_names(const lfr_plan* pl, uint32_t n_images, const uint8_t* names, const uint64_t* name_off, const char* missing,
                const uint32_t* group = nullptr, uint32_t G = 0) {
  if (!pl || !pl->graph) return fail(LFR_EINVAL, "plan was not made by lfr_plan_create_from_matches");
  if (n_images < pl->n_images) return fail(LFR_EINVAL, "n_images is smaller than the plan's image count");
  if (missing) return fail(LFR_EINVAL, missing);
  for (uint32_t k = 0; k < n_images; ++k) {
    if (name_off[k + 1] < name_off[k]) return fail(LFR_EINVAL, "name_off is not ascending");
    if (group && group[k] >= G) return fail(LFR_EINVAL, "an image's group is not below n_groups");
  }
  if (n_images && name_off[n_images] && !names) return fail(LFR_EINVAL, "names is NULL");
  return LFR_OK;
}

// What an lfr_plan_encode_solution* call encodes: the scene's image names and facts; optionally a group per
// image (one of G; G or more: the image is not written); optionally an earlier SolutionFile to carry, its
// bytes and their decode (G = 1 only).
struct EncodeInput {
  uint32_t n_images;
  const uint8_t* names;
  const uint64_t* name_off;
  const float* fact;
  const uint32_t* group = nullptr;
  uint32_t G = 1;
  const uint8_t* file = nullptr;
  const lfr::join::Decoded* decoded = nullptr;
};

// Every lfr_plan_encode_solution* call on a checked plan and input (lfr_solution.cuh): the sizing kernels
// (with a file, one synchronisation for the carried count among them), one synchronisation for the sizes,
// then, when `out` has room, the writing kernels, one synchronisation and one copy to `out`.  Host outputs:
// group_off[0..G], n_outside[0..G] (slot G: the images not written) and *n_carried.
int64_t encode_solution(lfr_plan* pl, cudaStream_t s, const EncodeInput& in, uint8_t* out, uint64_t cap,
                        uint64_t* group_off, uint64_t* n_outside, uint64_t* n_carried) {
  using namespace lfr::solution;
  const lfr::join::Decoded* d = in.decoded;
  assert(!d || in.G == 1);  // no call carries a file into several groups
  const uint32_t N = pl->N, NI = in.n_images, G = in.G;
  const uint32_t D = d ? (uint32_t)d->n_disp : 0, I = d ? (uint32_t)d->n_images : 0;
  std::fill(group_off, group_off + G + 1, 0);
  std::fill(n_outside, n_outside + G + 1, 0);
  *n_carried = 0;
  if (!N && !d) return 0;
  const auto t0 = Clock::now();
  // per message of the file: its key image (the scene id of a matched winner, NI + j for the j-th other
  // winner, kNoImage for a message that loses to a later one of its name), and the winners' names
  std::vector<uint32_t> msg_pid(I, kNoImage);
  std::vector<uint64_t> msg_name_off((size_t)I + 1, 0);
  std::vector<uint8_t> msg_names;
  uint64_t n_other = 0;
  for (uint32_t i = 0; i < I; ++i) {
    if (d->wins[i]) {
      msg_pid[i] = d->image_id[i] != lfr::join::kNoImage ? d->image_id[i] : (uint32_t)(NI + n_other++);
      msg_names.insert(msg_names.end(), in.file + d->name_off[i], in.file + d->name_off[i] + d->name_len[i]);
    }
    msg_name_off[(size_t)i + 1] = msg_names.size();
  }
  if ((uint64_t)NI + n_other >= kNoImage) return fail(LFR_EUNSUPPORTED, "too many images in the scene and the SolutionFile");
  const uint64_t name_bytes = in.name_off[NI];
  const uint32_t n_max = NI + I;  // an upper bound of the output images
  // an image's key: group << shift | its first node; an absent image's sorts after every group's images
  const int shift = bits_for(N);
  const unsigned long long absent = (unsigned long long)G << shift | N;

  unsigned long long *d_outside, *key, *key_s, *ekey, *ekey_s;
  uint32_t *n_present, *iota_i, *img_s, *rank, *d_group, *mpid, *g2, *g2_off, *g2_msg, *feat, *idx, *idx_s, *flag, *slot,
      *ce, *cm, *rkey, *rkey_s, *riota, *perm, *img_ptr;
  uint64_t *d_name_off, *mptr, *mnoff, *rsize, *roff, *body, *isize, *ioff, *goff;
  float *d_fact, *mfact, *di, *dj;
  uint8_t *d_names, *mnames, *used;
  // per scene image, per message, per entry, per record (N + at most D) and per output image
  LFR_TRY(carve(pl->enc_scratch, [&](Carve& c) {
    d_outside = c.take<unsigned long long>((size_t)G + 2);  // then n_present and n_out
    key = c.take<unsigned long long>(NI);
    key_s = c.take<unsigned long long>(NI);
    iota_i = c.take<uint32_t>(NI);
    img_s = c.take<uint32_t>(NI);
    rank = c.take<uint32_t>(NI);
    d_name_off = c.take<uint64_t>((size_t)NI + 1);
    d_fact = c.take<float>(NI);
    d_names = c.take<uint8_t>(name_bytes);
    d_group = c.take<uint32_t>(in.group ? NI : 0);
    mptr = c.take<uint64_t>((size_t)I + 1);
    mpid = c.take<uint32_t>(I);
    mnoff = c.take<uint64_t>((size_t)I + 1);
    mfact = c.take<float>(I);
    mnames = c.take<uint8_t>(msg_names.size());
    g2 = c.take<uint32_t>((size_t)I + 1);
    g2_off = c.take<uint32_t>((size_t)I + 1);
    g2_msg = c.take<uint32_t>(I);
    feat = c.take<uint32_t>(D);
    di = c.take<float>(D);
    dj = c.take<float>(D);
    ekey = c.take<unsigned long long>(D);
    ekey_s = c.take<unsigned long long>(D);
    idx = c.take<uint32_t>(D);
    idx_s = c.take<uint32_t>(D);
    used = c.take<uint8_t>(D);
    flag = c.take<uint32_t>((size_t)D + 1);
    slot = c.take<uint32_t>((size_t)D + 1);
    ce = c.take<uint32_t>(D);
    cm = c.take<uint32_t>(D);
    rkey = c.take<uint32_t>((size_t)N + D);
    rkey_s = c.take<uint32_t>((size_t)N + D);
    riota = c.take<uint32_t>((size_t)N + D);
    perm = c.take<uint32_t>((size_t)N + D);
    rsize = c.take<uint64_t>((size_t)N + D + 1);
    roff = c.take<uint64_t>((size_t)N + D + 1);
    img_ptr = c.take<uint32_t>((size_t)n_max + 1);
    body = c.take<uint64_t>(n_max);
    isize = c.take<uint64_t>((size_t)n_max + 1);
    ioff = c.take<uint64_t>((size_t)n_max + 1);
    goff = c.take<uint64_t>((size_t)G + 1);
  }));
  n_present = reinterpret_cast<uint32_t*>(d_outside + G + 1);
  uint32_t* n_out = d ? n_present + 1 : n_present;  // the output images: the present ones, then the file's others
  if (!in.group) d_group = nullptr;
  const uint32_t* nimg = pl->node_image.as<uint32_t>();
  const double* pos = pl->pos.as<double>();

  LFR_CUDA(cudaMemsetAsync(d_outside, 0, 8 * ((size_t)G + 2), s));
  LFR_CUDA(cudaMemcpyAsync(d_name_off, in.name_off, 8 * ((size_t)NI + 1), cudaMemcpyHostToDevice, s));
  if (NI) LFR_CUDA(cudaMemcpyAsync(d_fact, in.fact, 4 * (size_t)NI, cudaMemcpyHostToDevice, s));
  if (name_bytes) LFR_CUDA(cudaMemcpyAsync(d_names, in.names, name_bytes, cudaMemcpyHostToDevice, s));
  if (d_group && NI) LFR_CUDA(cudaMemcpyAsync(d_group, in.group, 4 * (size_t)NI, cudaMemcpyHostToDevice, s));
  // the present images, ranked by (group, first node)
  if (NI) {
    init_images_kernel<<<blocks_for(NI), 256, 0, s>>>(key, iota_i, NI, absent);
    if (N) first_node_kernel<<<blocks_for(N), 256, 0, s>>>(nimg, pos, N, d_group, G, shift, key, d_outside);
    LFR_LAUNCHED();
    LFR_TRY(cub_run(pl->enc_cub, [&](void* t, size_t& nb) {
      return cub::DeviceRadixSort::SortPairs(t, nb, key, key_s, iota_i, img_s, (int)NI, 0, shift + bits_for(G), s);
    }));
    rank_kernel<<<blocks_for(NI), 256, 0, s>>>(key_s, img_s, NI, absent, rank, n_present);
    LFR_LAUNCHED();
  }
  // the file's entries: keyed, sorted stably, joined to the nodes, the carried ones compacted; its other
  // winning messages ranked after the present scene images in file order
  uint32_t C = 0;
  if (d) {
    LFR_CUDA(cudaMemcpyAsync(mptr, d->img_ptr.data(), 8 * ((size_t)I + 1), cudaMemcpyHostToDevice, s));
    LFR_CUDA(cudaMemcpyAsync(mnoff, msg_name_off.data(), 8 * ((size_t)I + 1), cudaMemcpyHostToDevice, s));
    if (I) {
      LFR_CUDA(cudaMemcpyAsync(mpid, msg_pid.data(), 4 * (size_t)I, cudaMemcpyHostToDevice, s));
      LFR_CUDA(cudaMemcpyAsync(mfact, d->fact.data(), 4 * (size_t)I, cudaMemcpyHostToDevice, s));
    }
    if (!msg_names.empty()) LFR_CUDA(cudaMemcpyAsync(mnames, msg_names.data(), msg_names.size(), cudaMemcpyHostToDevice, s));
    if (D) {
      LFR_CUDA(cudaMemcpyAsync(feat, d->feature_idx.data(), 4 * (size_t)D, cudaMemcpyHostToDevice, s));
      LFR_CUDA(cudaMemcpyAsync(di, d->di.data(), 4 * (size_t)D, cudaMemcpyHostToDevice, s));
      LFR_CUDA(cudaMemcpyAsync(dj, d->dj.data(), 4 * (size_t)D, cudaMemcpyHostToDevice, s));
      LFR_CUDA(cudaMemsetAsync(used, 0, D, s));
      lfr::start::solution_key_kernel<<<blocks_for(D), 256, 0, s>>>(mptr, mpid, I, feat, D, ekey, idx);
      LFR_LAUNCHED();
      LFR_TRY(cub_run(pl->enc_cub, [&](void* t, size_t& nb) {  // stable: equal keys stay in file order
        return cub::DeviceRadixSort::SortPairs(t, nb, ekey, ekey_s, idx, idx_s, (int)D, 0, 64, s);
      }));
      if (N) consume_kernel<<<blocks_for(N), 256, 0, s>>>(nimg, pl->node_feat.as<uint32_t>(), N, ekey_s, D, used);
      carry_flag_kernel<<<blocks_for((uint64_t)D + 1), 256, 0, s>>>(ekey_s, used, D, flag);
      LFR_LAUNCHED();
      LFR_TRY(cub_run(pl->enc_cub, [&](void* t, size_t& nb) { return cub::DeviceScan::ExclusiveSum(t, nb, flag, slot, (int)D + 1, s); }));
      carry_compact_kernel<<<blocks_for(D), 256, 0, s>>>(flag, slot, idx_s, mptr, I, D, ce, cm);
      LFR_LAUNCHED();
      LFR_TRY(fetch(&C, slot + D, 1, s));
    }
    group2_flag_kernel<<<blocks_for((uint64_t)I + 1), 256, 0, s>>>(mpid, I, key, NI, absent, g2);
    LFR_LAUNCHED();
    LFR_TRY(cub_run(pl->enc_cub, [&](void* t, size_t& nb) { return cub::DeviceScan::ExclusiveSum(t, nb, g2, g2_off, (int)I + 1, s); }));
    group2_scatter_kernel<<<blocks_for((uint64_t)I + 1), 256, 0, s>>>(g2, g2_off, I, n_present, g2_msg, n_out);
    LFR_LAUNCHED();
  }
  // the records (nodes, then carried entries) in output order, their sizes and the images'
  const uint32_t R = N + C;
  const Records rec{N, pl->node_feat.as<uint32_t>(), pos, ce, feat, di, dj};
  const Headers hdr{n_present, img_s, d_names, d_name_off, d_fact, g2_msg, mnames, mnoff, mfact};
  if (R) {
    record_key_kernel<<<blocks_for(R), 256, 0, s>>>(nimg, d_group, G, rank, N, cm, mpid, g2, g2_off, n_present, R, n_max,
                                                     rkey, riota);
    LFR_LAUNCHED();
    LFR_TRY(cub_run(pl->enc_cub, [&](void* t, size_t& nb) {  // stable: nodes by index, then carried entries by feature
      return cub::DeviceRadixSort::SortPairs(t, nb, rkey, rkey_s, riota, perm, (int)R, 0, bits_for(n_max), s);
    }));
  }
  record_size_kernel<<<blocks_for((uint64_t)R + 1), 256, 0, s>>>(perm, rkey_s, R, rec, n_out, rsize, img_ptr);
  LFR_LAUNCHED();
  LFR_TRY(cub_run(pl->enc_cub, [&](void* t, size_t& nb) { return cub::DeviceScan::ExclusiveSum(t, nb, rsize, roff, (int)R + 1, s); }));
  image_size_kernel<<<blocks_for((uint64_t)n_max + 1), 256, 0, s>>>(hdr, img_ptr, roff, n_out, n_max, body, isize);
  LFR_LAUNCHED();
  LFR_TRY(cub_run(pl->enc_cub, [&](void* t, size_t& nb) { return cub::DeviceScan::ExclusiveSum(t, nb, isize, ioff, (int)n_max + 1, s); }));
  // one group: {0, the total}
  if (G > 1) {
    group_off_kernel<<<blocks_for((uint64_t)NI + 1), 256, 0, s>>>(key_s, NI, shift, G, ioff, goff);
    LFR_LAUNCHED();
  }
  LFR_CUDA(cudaMemcpyAsync(n_outside, d_outside, 8 * ((size_t)G + 1), cudaMemcpyDeviceToHost, s));
  LFR_TRY(G > 1 ? fetch(group_off, goff, (size_t)G + 1, s) : fetch(group_off + 1, ioff + n_max, 1, s));
  const uint64_t total = group_off[G];
  *n_carried = C;
  if (!out || cap < total || !total) return (int64_t)total;
  LFR_TRY(pl->enc_out.reserve(total));
  uint8_t* d_out = pl->enc_out.as<uint8_t>();
  if (n_max) write_images_kernel<<<blocks_for(n_max), 256, 0, s>>>(hdr, body, ioff, n_out, n_max, d_out);
  if (R) write_records_kernel<<<blocks_for(R), 256, 0, s>>>(perm, rkey_s, R, rec, img_ptr, roff, ioff, n_out, d_out);
  LFR_LAUNCHED();
  LFR_CUDA(cudaStreamSynchronize(s));
  g_encode_ms[0] = ms_since(t0);
  const auto t1 = Clock::now();
  LFR_TRY(fetch(out, d_out, total, s));
  g_encode_ms[1] = ms_since(t1);
  return (int64_t)total;
}

// encode_solution() for the calls with one output: its "> 0.5" count summed over the slots
int64_t encode_one(lfr_plan* pl, void* stream, const EncodeInput& in, uint8_t* out, uint64_t cap, uint64_t* n_outside,
                   uint64_t* n_carried = nullptr) {
  uint64_t group_off[2], outside[2], carried;
  const int64_t total = encode_solution(pl, (cudaStream_t)stream, in, out, cap, group_off, outside, &carried);
  if (n_outside) *n_outside = outside[0] + outside[1];
  if (n_carried) *n_carried = carried;
  return total;
}

int select_device(const lfr_options& o) {
  int n_dev = 0;
  LFR_CUDA(cudaGetDeviceCount(&n_dev));
  if (n_dev == 0) return fail(LFR_ENODEV, "no CUDA device");
  if (o.device < 0 || o.device >= n_dev) return fail(LFR_ENODEV, "device ordinal out of range");
  LFR_CUDA(cudaSetDevice(o.device));
  return LFR_OK;
}

// lfr_solve()'s workspace: per device (shared by all host threads, guarded by g_ws_mutex), one cached
// plan (grow-only device buffers), one non-blocking stream and the events that time the call — all
// created with that device current.  Kept until lfr_shutdown() or process exit (no destructor calls
// into CUDA during teardown).
struct DeviceWorkspace {
  lfr_plan* plan = nullptr;
  cudaStream_t stream = nullptr;
  cudaEvent_t ev[4] = {};
  bool ready = false;
};
constexpr int kMaxDevices = 16;
DeviceWorkspace g_ws[kMaxDevices];
std::mutex g_ws_mutex[kMaxDevices];  // one solve at a time per device workspace; distinct devices run concurrently

int ensure_workspace(int device) {
  DeviceWorkspace& ws = g_ws[device];
  if (ws.ready) return LFR_OK;
  LFR_CUDA(cudaStreamCreateWithFlags(&ws.stream, cudaStreamNonBlocking));
  for (int i = 0; i < 4; ++i) LFR_CUDA(cudaEventCreate(&ws.ev[i]));
  ws.plan = new lfr_plan();
  ws.plan->device = device;
  ws.ready = true;
  return LFR_OK;
}

// One device's part of a solve: uploads, launches, results.  `slot_owner` / `owner_id` restrict the
// plan to the dispatch slots this device owns (nullptr = all).  `in_place`: page-locked caller buffers
// are read / written where they are (zero-copy) instead of going through HBM.  Caller holds
// g_ws_mutex[device].
int solve_on_device(const lfr_problem* p, const lfr_options& o, double* positions, lfr_stats* st,
                    const uint8_t* slot_owner, uint8_t owner_id, double* pos_scratch, bool in_place) {
  LFR_TRY(select_device(o));
  LFR_TRY(ensure_workspace(o.device));
  DeviceWorkspace& ws = g_ws[o.device];
  lfr_plan* pl = ws.plan;
  cudaStream_t s = ws.stream;
  pl->slot_owner = slot_owner;
  pl->owner_id = owner_id;
  // page-locked caller buffers are used in place only where the caller asked for it (see include/lfr.h)
  const bool zero_copy = in_place && !(o.debug_flags & LFR_DBG_NO_ZERO_COPY);
  const float4* zc_edges = (zero_copy && p->n_edges) ? static_cast<const float4*>(device_view_of_pinned(p->edges)) : nullptr;
  double* zc_positions = (zero_copy && p->n_nodes) ? static_cast<double*>(device_view_of_pinned(positions)) : nullptr;
  g_host_t0 = std::chrono::steady_clock::now();
  LFR_CUDA(cudaEventRecord(ws.ev[0], s));
  LFR_TRY(fill_plan(pl, p, o, positions, s, /*stage_positions_directly=*/true, zc_edges, zc_positions));
  host_mark(2);
  LFR_CUDA(cudaEventRecord(ws.ev[1], s));
  LFR_TRY(launch_solve(pl, s));
  LFR_CUDA(cudaEventRecord(ws.ev[2], s));
  host_mark(3);
  // several devices, pageable positions: each device returns its copy into its own scratch array
  // and the caller merges the entries of the components it owns
  int rc = download(pl, s, (slot_owner && !zc_positions) ? pos_scratch : positions, st);
  if (pl->copy_stream && pl->zc_edges && pl->edges_in_hbm) {
    // the bulk copy reads the caller's buffer: it must be over before the call returns
    cudaError_t e = cudaStreamSynchronize(pl->copy_stream);
    if (e != cudaSuccess && rc == LFR_OK) rc = fail(cuda_code(e), cudaGetErrorString(e));
  }
  host_mark(4);
  pl->slot_owner = nullptr;
  if (rc) return rc;
  LFR_CUDA(cudaEventRecord(ws.ev[3], s));
  LFR_CUDA(cudaEventSynchronize(ws.ev[3]));
  host_mark(5);
  if (st) {
    float a = 0, b = 0, c = 0;
    cudaEventElapsedTime(&a, ws.ev[0], ws.ev[1]);
    cudaEventElapsedTime(&b, ws.ev[1], ws.ev[2]);
    cudaEventElapsedTime(&c, ws.ev[2], ws.ev[3]);
    st->h2d_ms = a;     // uploads of the arrays that go through HBM (+ schedule)
    st->kernel_ms = b;  // the solve kernels (with zero-copy: including their PCIe pulls)
    st->d2h_ms = c;
    st->total_ms = (double)a + b + c;
  }
  return LFR_OK;
}

// The constant mask of a plan made from matches (reference root OR node of a fixed image OR kept node),
// expanded on the device over the plan's node ids, and the schedule built again on it: free-node counts
// move components between tiers.  Synchronous on `s`.
int build_constant_mask(lfr_plan* pl, cudaStream_t s) {
  const lfr_plan::GraphArrays& G = *pl->graph;
  const uint32_t N = pl->N;
  LFR_TRY(pl->const_mask.reserve(std::max<size_t>(N, 1)));
  if (N) {
    const uint8_t* fixed = nullptr;
    if (!pl->fixed_host.empty()) {
      LFR_TRY(upload(&pl->enc_scratch, pl->fixed_host.data(), pl->fixed_host.size(), s));
      fixed = pl->enc_scratch.as<uint8_t>();
    }
    lfr::start::constant_mask_kernel<<<blocks_for(N), 256, 0, s>>>(pl->is_root.as<uint8_t>(), pl->node_image.as<uint32_t>(),
                                                                     fixed, pl->kept.p ? pl->kept.as<uint8_t>() : nullptr,
                                                                     N, pl->const_mask.as<uint8_t>());
    LFR_LAUNCHED();
  }
  pl->const_host.resize(N);
  LFR_TRY(fetch(pl->const_host.data(), pl->const_mask.p, N, s));
  lfr_problem p;
  p.n_nodes = N;
  p.n_components = pl->C;
  p.n_edges = pl->E;
  p.row_ptr = G.row_ptr.data();
  p.edges = nullptr;  // in pl->edges
  p.track = G.track.data();
  p.comp = G.comp.data();
  p.is_root = pl->const_host.data();
  p.comp_ptr = G.comp_ptr.data();
  p.comp_nodes = G.comp_nodes.data();
  LFR_TRY(schedule_plan(pl, &p, s));
  LFR_CUDA(cudaStreamSynchronize(s));
  return LFR_OK;
}

// The arguments of lfr_plan_start_from_solution / lfr_plan_keep_solution checked, and the SolutionFile
// decoded and its images resolved on the host (lfr_join.h), before either call changes the plan.
int decode_solution_for(const lfr_plan* pl, const uint8_t* bytes, uint64_t len, uint32_t n_images, const uint8_t* names,
                        const uint64_t* name_off, lfr::join::Decoded& d) {
  LFR_TRY(check_names(pl, n_images, names, name_off,
                      (len && !bytes) || (n_images && !name_off) ? "NULL SolutionFile bytes or image names" : nullptr));
  const uint8_t no_name = 0;
  if (lfr::join::decode(bytes, len, n_images, names ? names : &no_name, name_off, d) != LFR_OK)
    return fail(LFR_EINVAL, "malformed SolutionFile");
  if (d.n_disp >= (1ull << 31)) return fail(LFR_EUNSUPPORTED, "SolutionFile with 2^31 or more displacements");
  return LFR_OK;
}

// The device join of a decoded SolutionFile against the plan's nodes: writes the start and working
// positions, and has_entry[v] when it is not NULL.
int join_solution(lfr_plan* pl, cudaStream_t s, const lfr::join::Decoded& d, uint8_t* has_entry, uint64_t* n_started) {
  const uint32_t N = pl->N, D = (uint32_t)d.n_disp, I = (uint32_t)d.n_images;
  if (n_started) *n_started = 0;
  if (!N) return LFR_OK;
  unsigned long long *ctr, *key, *key_s;
  uint64_t* img_ptr;
  uint32_t *image_id, *feat, *idx, *idx_s;
  float *di, *dj;
  LFR_TRY(carve(pl->enc_scratch, [&](Carve& c) {
    ctr = c.take<unsigned long long>(1);
    img_ptr = c.take<uint64_t>((size_t)I + 1);
    image_id = c.take<uint32_t>((size_t)I + 1);
    feat = c.take<uint32_t>(D);
    di = c.take<float>(D);
    dj = c.take<float>(D);
    key = c.take<unsigned long long>(D);
    key_s = c.take<unsigned long long>(D);
    idx = c.take<uint32_t>(D);
    idx_s = c.take<uint32_t>(D);
  }));
  LFR_CUDA(cudaMemsetAsync(ctr, 0, 8, s));
  if (D) {
    LFR_CUDA(cudaMemcpyAsync(img_ptr, d.img_ptr.data(), 8 * ((size_t)I + 1), cudaMemcpyHostToDevice, s));
    LFR_CUDA(cudaMemcpyAsync(image_id, d.image_id.data(), 4 * (size_t)I, cudaMemcpyHostToDevice, s));
    LFR_CUDA(cudaMemcpyAsync(feat, d.feature_idx.data(), 4 * (size_t)D, cudaMemcpyHostToDevice, s));
    LFR_CUDA(cudaMemcpyAsync(di, d.di.data(), 4 * (size_t)D, cudaMemcpyHostToDevice, s));
    LFR_CUDA(cudaMemcpyAsync(dj, d.dj.data(), 4 * (size_t)D, cudaMemcpyHostToDevice, s));
    lfr::start::solution_key_kernel<<<blocks_for(D), 256, 0, s>>>(img_ptr, image_id, I, feat, D, key, idx);
    LFR_LAUNCHED();
    LFR_TRY(cub_run(pl->enc_cub, [&](void* t, size_t& nb) {  // stable: equal keys stay in file order
      return cub::DeviceRadixSort::SortPairs(t, nb, key, key_s, idx, idx_s, (int)D, 0, 64, s);
    }));
  }
  // image ids that share a name join through the lowest of them (lfr_join.h): the nodes keyed by that id
  const uint32_t* node_image = pl->node_image.as<uint32_t>();
  TmpBuf d_canon, d_nkey;
  if (!d.canon.empty()) {
    LFR_TRY(upload(&d_canon, d.canon.data(), d.canon.size(), s));
    LFR_TRY(d_nkey.reserve(4 * (size_t)N));
    lfr::graph::gather_kernel<<<blocks_for(N), 256, 0, s>>>(node_image, d_canon.as<uint32_t>(), N, d_nkey.as<uint32_t>());
    LFR_LAUNCHED();
    node_image = d_nkey.as<uint32_t>();
  }
  lfr::start::join_kernel<<<blocks_for(N), 256, 0, s>>>(node_image, pl->node_feat.as<uint32_t>(), N,
                                                          key_s, idx_s, D, di, dj, pl->pos_init.as<double>(),
                                                          pl->pos.as<double>(), ctr, has_entry);
  LFR_LAUNCHED();
  pl->pos_is_staged = true;  // the working positions hold the new start point (as after creation)
  unsigned long long started = 0;
  LFR_TRY(fetch(&started, ctr, 1, s));  // also keeps `d` alive until its copies are done
  if (n_started) *n_started = started;
  return LFR_OK;
}

// lfr_plan_update_solution() after the decode, with the touched flags seeded from changed[C] on the device
// (NULL: none; lfr_plan_update_solution_since)
int update_solution(lfr_plan* pl, cudaStream_t s, const lfr::join::Decoded& d, const uint8_t* changed, uint64_t* n_held,
                    uint32_t* n_touched) {
  const uint32_t N = pl->N, C = pl->C;
  if (!pl->kept.p) {  // cleared, so that a join that fails before its kernel leaves no stale flags
    LFR_TRY(pl->kept.reserve(std::max<size_t>(N, 1)));
    LFR_CUDA(cudaMemsetAsync(pl->kept.p, 0, std::max<size_t>(N, 1), s));
  }
  // the kept flags take the join's "has entry", then the held flags in place
  LFR_TRY(join_solution(pl, s, d, pl->kept.as<uint8_t>(), nullptr));
  unsigned long long counts[2] = {0, 0};  // held nodes, touched components
  if (N) {
    TmpBuf t;  // the two counters, then one touched flag per component
    LFR_TRY(t.reserve(16 + (size_t)C));
    auto* ctr = t.as<unsigned long long>();
    uint8_t* touched = t.as<uint8_t>() + 16;
    LFR_CUDA(cudaMemsetAsync(t.p, 0, 16 + (size_t)C, s));
    if (changed && C) LFR_CUDA(cudaMemcpyAsync(touched, changed, C, cudaMemcpyDeviceToDevice, s));
    lfr::start::touch_kernel<<<blocks_for(N), 256, 0, s>>>(pl->kept.as<uint8_t>(), pl->comp.as<uint32_t>(), N, touched);
    lfr::start::update_kernel<<<blocks_for(N), 256, 0, s>>>(pl->comp.as<uint32_t>(), touched, N, pl->kept.as<uint8_t>(),
                                                              pl->pos_init.as<double>(), pl->pos.as<double>(), ctr);
    lfr::start::count_touched_kernel<<<blocks_for(C), 256, 0, s>>>(touched, C, ctr + 1);
    LFR_LAUNCHED();
    LFR_TRY(fetch(counts, ctr, 2, s));  // before `t` is freed
  }
  if (n_held) *n_held = counts[0];
  if (n_touched) *n_touched = (uint32_t)counts[1];
  return build_constant_mask(pl, s);
}

// lfr_plan_update_solution_since(): changed[c] = 1 (device, C flags) for every component c of `pl` that fails
// the "unchanged" test against `prev` (lfr_diff.cuh); `image_map` (host, prev's image count) gives prev's image
// ids in pl's numbering.  *n_changed = the count.  Reads both plans, changes neither.
int diff_components(const lfr_plan* pl, const lfr_plan* prev, const std::vector<uint32_t>& image_map, cudaStream_t s,
                    uint8_t* changed, uint32_t* n_changed) {
  using namespace lfr::diff;
  const uint32_t N = pl->N, C = pl->C, M = prev->N, PC = prev->C;
  const uint64_t E = pl->E, EB = prev->E, R = E + EB;
  LFR_CUDA(cudaMemsetAsync(changed, 0, std::max<size_t>(C, 1), s));
  *n_changed = 0;
  if (!N) return LFR_OK;
  if (R >= (1ull << 31)) return fail(LFR_EUNSUPPORTED, "2^31 or more directed edges in the two plans");
  TmpBuf tmp, d_map, d_key, d_key_s, d_idx, d_idx_s, d_inv, d_lo, d_hi, d_size, d_psize, d_ekey, d_ekey_s, d_eval, d_eval_s, d_ctr;
  LFR_TRY(d_map.reserve(4 * std::max<size_t>(image_map.size(), 1)));
  for (TmpBuf* b : {&d_key, &d_key_s}) LFR_TRY(b->reserve(8 * std::max<size_t>(M, 1)));
  for (TmpBuf* b : {&d_idx, &d_idx_s, &d_inv}) LFR_TRY(b->reserve(4 * std::max<size_t>(M, 1)));
  for (TmpBuf* b : {&d_lo, &d_hi, &d_size}) LFR_TRY(b->reserve(4 * (size_t)C));
  LFR_TRY(d_psize.reserve(4 * std::max<size_t>(PC, 1)));
  for (TmpBuf* b : {&d_ekey, &d_ekey_s, &d_eval, &d_eval_s}) LFR_TRY(b->reserve(8 * std::max<size_t>(R, 1)));
  LFR_TRY(d_ctr.reserve(8));
  auto* key = d_key.as<unsigned long long>();
  auto* key_s = d_key_s.as<unsigned long long>();
  auto* lo = d_lo.as<uint32_t>();
  auto* hi = d_hi.as<uint32_t>();
  auto* size = d_size.as<uint32_t>();
  auto* psize = d_psize.as<uint32_t>();
  auto* inv = d_inv.as<uint32_t>();
  if (!image_map.empty())
    LFR_CUDA(cudaMemcpyAsync(d_map.p, image_map.data(), 4 * image_map.size(), cudaMemcpyHostToDevice, s));
  LFR_CUDA(cudaMemsetAsync(lo, 0xff, 4 * (size_t)C, s));
  LFR_CUDA(cudaMemsetAsync(hi, 0, 4 * (size_t)C, s));
  LFR_CUDA(cudaMemsetAsync(size, 0, 4 * (size_t)C, s));
  LFR_CUDA(cudaMemsetAsync(psize, 0, 4 * std::max<size_t>(PC, 1), s));
  LFR_CUDA(cudaMemsetAsync(inv, 0xff, 4 * std::max<size_t>(M, 1), s));
  LFR_CUDA(cudaMemsetAsync(d_ctr.p, 0, 8, s));
  if (M) {
    prev_key_kernel<<<blocks_for(M), 256, 0, s>>>(prev->node_image.as<uint32_t>(), prev->node_feat.as<uint32_t>(), M,
                                                  d_map.as<uint32_t>(), key, d_idx.as<uint32_t>());
    LFR_LAUNCHED();
    LFR_TRY(cub_run(tmp, [&](void* t, size_t& nb) {  // keys are distinct: the mapped names are
      return cub::DeviceRadixSort::SortPairs(t, nb, key, key_s, d_idx.as<uint32_t>(), d_idx_s.as<uint32_t>(), (int)M, 0, 64, s);
    }));
    size_kernel<<<blocks_for(M), 256, 0, s>>>(prev->comp.as<uint32_t>(), M, psize);
    LFR_LAUNCHED();
  }
  node_kernel<<<blocks_for(N), 256, 0, s>>>(pl->node_image.as<uint32_t>(), pl->node_feat.as<uint32_t>(), pl->comp.as<uint32_t>(),
                                            pl->is_root.as<uint8_t>(), N, key_s, d_idx_s.as<uint32_t>(), M,
                                            prev->comp.as<uint32_t>(), prev->is_root.as<uint8_t>(), inv, lo, hi, size, changed);
  comp_kernel<<<blocks_for(C), 256, 0, s>>>(lo, hi, size, psize, C, changed);
  LFR_LAUNCHED();
  const unsigned long long sentinel = (unsigned long long)N << 32;
  auto* ekey = d_ekey.as<unsigned long long>();
  auto* eval = d_eval.as<unsigned long long>();
  if (E)
    edge_key_kernel<<<blocks_for(E), 256, 0, s>>>(pl->row_ptr.as<uint32_t>(), pl->edges.as<float4>(), pl->track.as<uint32_t>(),
                                                  pl->comp.as<uint32_t>(), N, (uint32_t)E, nullptr, 0ull, sentinel, ekey, eval);
  if (EB)
    edge_key_kernel<<<blocks_for(EB), 256, 0, s>>>(prev->row_ptr.as<uint32_t>(), prev->edges.as<float4>(),
                                                   prev->track.as<uint32_t>(), prev->comp.as<uint32_t>(), M, (uint32_t)EB, inv,
                                                   1ull, sentinel, ekey + E, eval + E);
  LFR_LAUNCHED();
  if (R) {
    LFR_TRY(cub_run(tmp, [&](void* t, size_t& nb) {
      return cub::DeviceRadixSort::SortPairs(t, nb, ekey, d_ekey_s.as<unsigned long long>(), eval,
                                             d_eval_s.as<unsigned long long>(), (int)R, 0, 32 + bits_for(N), s);
    }));
    run_kernel<<<blocks_for(R), 256, 0, s>>>(d_ekey_s.as<unsigned long long>(), d_eval_s.as<unsigned long long>(), (uint32_t)R,
                                             sentinel, pl->edges.as<uint32_t>(), prev->edges.as<uint32_t>(),
                                             pl->comp.as<uint32_t>(), changed);
    LFR_LAUNCHED();
  }
  lfr::start::count_touched_kernel<<<blocks_for(C), 256, 0, s>>>(changed, C, d_ctr.as<unsigned long long>());
  LFR_LAUNCHED();
  unsigned long long nc = 0;
  LFR_TRY(fetch(&nc, d_ctr.p, 1, s));  // before the scratch is freed
  *n_changed = (uint32_t)nc;
  return LFR_OK;
}

// The digest of every component of `pl` (lfr_record.cuh) into d0[C], d1[C] (device, reserved here): name ids
// hashed on the host, elements hashed and summed on the device.  Reads the plan, changes nothing.
int plan_digests(const lfr_plan* pl, cudaStream_t s, uint32_t n_images, const uint8_t* names, const uint64_t* name_off,
                 TmpBuf& d0, TmpBuf& d1) {
  const uint32_t N = pl->N, C = pl->C;
  const uint64_t E = pl->E;
  std::vector<unsigned long long> ids(2 * (size_t)std::max<uint32_t>(n_images, 1), 0);
  for (uint32_t k = 0; k < n_images; ++k) {
    uint64_t h0, h1;
    lfr::record::hash_bytes(names + name_off[k], name_off[k + 1] - name_off[k], h0, h1);
    ids[2 * (size_t)k] = h0;
    ids[2 * (size_t)k + 1] = h1;
  }
  LFR_TRY(d0.reserve(8 * std::max<size_t>(C, 1)));
  LFR_TRY(d1.reserve(8 * std::max<size_t>(C, 1)));
  if (!C) return LFR_OK;
  TmpBuf d_ids;
  LFR_TRY(d_ids.reserve(8 * ids.size()));
  LFR_CUDA(cudaMemcpyAsync(d_ids.p, ids.data(), 8 * ids.size(), cudaMemcpyHostToDevice, s));
  LFR_CUDA(cudaMemsetAsync(d0.p, 0, 8 * (size_t)C, s));
  LFR_CUDA(cudaMemsetAsync(d1.p, 0, 8 * (size_t)C, s));
  if (N + E) {
    lfr::record::digest_kernel<<<blocks_for(N + E), 256, 0, s>>>(
        pl->row_ptr.as<uint32_t>(), pl->edges.as<float4>(), pl->track.as<uint32_t>(), pl->comp.as<uint32_t>(),
        pl->is_root.as<uint8_t>(), pl->node_image.as<uint32_t>(), pl->node_feat.as<uint32_t>(), d_ids.as<ulonglong2>(), N,
        E, d0.as<unsigned long long>(), d1.as<unsigned long long>());
    LFR_LAUNCHED();
  }
  LFR_CUDA(cudaStreamSynchronize(s));  // before `d_ids` is freed
  return LFR_OK;
}

// The group of every component of `pl` into cgroup[C] (device, reserved here), from the caller's group of every
// image (uploaded into d_group, reserved here)
int component_groups(const lfr_plan* pl, cudaStream_t s, uint32_t n_images, const uint32_t* group_of_image, TmpBuf& d_group,
                     TmpBuf& cgroup) {
  const uint32_t N = pl->N, C = pl->C;
  LFR_TRY(upload(&d_group, group_of_image, n_images, s));
  LFR_TRY(cgroup.reserve(4 * std::max<size_t>(C, 1)));
  if (N) {
    lfr::record::component_group_kernel<<<blocks_for(N), 256, 0, s>>>(pl->comp.as<uint32_t>(), pl->node_image.as<uint32_t>(),
                                                                      d_group.as<uint32_t>(), N, cgroup.as<uint32_t>());
    LFR_LAUNCHED();
  }
  return LFR_OK;
}
}  // namespace

extern "C" {

int lfr_abi_version(void) { return LFR_ABI_VERSION; }
const char* lfr_backend(void) { return "b200"; }
const char* lfr_last_error(void) { return g_last_error.c_str(); }

void lfr_options_default(lfr_options* o) {
  if (!o) return;
  std::memset(o, 0, sizeof *o);
  o->bound = 1.0;                 // solve.cc:89
  o->cauchy_a = 0.25;             // solve.cc:111
  o->tukey_a = 0.0625;            // solve.cc:120
  o->tukey_variant = 1;
  o->max_num_iterations = 100;    // solve.cc:149
  o->max_num_consecutive_invalid_steps = 10;  // solve.cc:151
  o->max_num_line_search_step_size_iterations = 20;
  o->function_tolerance = 1e-4;   // solve.cc:152
  o->gradient_tolerance = 1e-8;   // solve.cc:153
  o->parameter_tolerance = 1e-4;  // solve.cc:154
  o->initial_trust_region_radius = 1e4;
  o->max_trust_region_radius = 1e16;
  o->min_trust_region_radius = 1e-32;
  o->min_relative_decrease = 1e-3;
  o->min_lm_diagonal = 1e-6;
  o->max_lm_diagonal = 1e32;
  o->line_search_sufficient_function_decrease = 1e-4;
  o->max_line_search_step_contraction = 1e-3;
  o->min_line_search_step_contraction = 0.6;
  o->min_line_search_step_size = 1e-9;
  o->n_threads = 8;
  o->device = 0;
  o->linear_solver = 0;
}

int lfr_plan_create(const lfr_problem* p, const lfr_options* opt, const double* initial_positions,
                    lfr_plan** out) {
  if (!out) return fail(LFR_EINVAL, "out is NULL");
  *out = nullptr;
  LFR_TRY(validate(p));
  lfr_options o;
  if (opt) o = *opt; else lfr_options_default(&o);
  LFR_TRY(select_device(o));
  lfr_plan* pl = new lfr_plan();
  pl->device = o.device;
  int rc = fill_plan(pl, p, o, initial_positions, 0);
  if (rc == LFR_OK) {
    cudaError_t e = cudaStreamSynchronize(0);
    if (e != cudaSuccess) rc = fail(cuda_code(e), cudaGetErrorString(e));
  }
  if (rc) {
    free_plan(pl);
    return rc;
  }
  *out = pl;
  return LFR_OK;
}

int lfr_plan_create_from_matches(const lfr_host_input* in, const lfr_options* opt, const double* initial_positions,
                                 lfr_plan** out, lfr_host_sizes* sizes) {
  if (!out) return fail(LFR_EINVAL, "out is NULL");
  *out = nullptr;
  if (!in) return fail(LFR_EINVAL, "input is NULL");
  lfr_options o;
  if (opt) o = *opt; else lfr_options_default(&o);
  LFR_TRY(select_device(o));
  lfr_plan* pl = new lfr_plan();
  pl->device = o.device;
  lfr_host_sizes S;
  MatchArrays d;
  int rc = upload_matches(in, d, 0);
  if (rc == LFR_OK) rc = create_plan_from_graph(in, d, o, initial_positions, pl, &S);
  if (rc) {
    free_plan(pl);
    return rc;
  }
  if (sizes) *sizes = S;
  *out = pl;
  return LFR_OK;
}

int lfr_plan_create_from_wire(const lfr_host_input* in, const lfr_wire_part* parts, uint32_t n_parts,
                              const lfr_options* opt, const double* initial_positions, lfr_plan** out,
                              lfr_host_sizes* sizes) {
  if (!out) return fail(LFR_EINVAL, "out is NULL");
  *out = nullptr;
  if (!in) return fail(LFR_EINVAL, "input is NULL");
  if (n_parts && !parts) return fail(LFR_EINVAL, "parts is NULL");
  lfr_options o;
  if (opt) o = *opt; else lfr_options_default(&o);
  LFR_TRY(select_device(o));
  lfr_plan* pl = new lfr_plan();
  pl->device = o.device;
  lfr_host_sizes S;
  MatchArrays d;
  int rc = decode_wire_on_device(in, parts, n_parts, d, 0);
  if (rc == LFR_OK) rc = create_plan_from_graph(in, d, o, initial_positions, pl, &S);
  if (rc) {
    free_plan(pl);
    return rc;
  }
  if (sizes) *sizes = S;
  *out = pl;
  return LFR_OK;
}

int lfr_plan_create_from_wire_listed(const lfr_host_input* in, const lfr_wire_part* parts, uint32_t n_parts,
                                     const uint64_t* src_pair_ptr, uint64_t n_src_pairs, const uint64_t* pair_src,
                                     const lfr_options* opt, const double* initial_positions, lfr_plan** out,
                                     lfr_host_sizes* sizes) {
  if (!out) return fail(LFR_EINVAL, "out is NULL");
  *out = nullptr;
  if (!in) return fail(LFR_EINVAL, "input is NULL");
  if (n_parts && !parts) return fail(LFR_EINVAL, "parts is NULL");
  if (!src_pair_ptr || (in->n_pairs && (!pair_src || !in->pair_ptr)))
    return fail(LFR_EINVAL, "NULL src_pair_ptr, pair_src or pair_ptr");
  // the entries against the file's pair level: every source pair exists, and in->pair_ptr is the scan of
  // the entries' match counts (the stage reads it on the host; the expand computes it on the device)
  if (src_pair_ptr[0] != 0) return fail(LFR_EINVAL, "src_pair_ptr[0] is not 0");
  for (uint64_t p = 0; p < n_src_pairs; ++p)
    if (src_pair_ptr[p + 1] < src_pair_ptr[p]) return fail(LFR_EINVAL, "src_pair_ptr decreases");
  if (in->n_pairs && in->pair_ptr[0] != 0) return fail(LFR_EINVAL, "pair_ptr[0] is not 0");
  for (uint64_t k = 0; k < in->n_pairs; ++k) {
    if (pair_src[k] >= n_src_pairs) return fail(LFR_EINVAL, "a listed pair's source is out of range");
    if (in->pair_ptr[k + 1] - in->pair_ptr[k] != src_pair_ptr[pair_src[k] + 1] - src_pair_ptr[pair_src[k]])
      return fail(LFR_EINVAL, "pair_ptr is not the scan of the listed pairs' match counts");
  }
  if ((in->n_pairs ? in->pair_ptr[in->n_pairs] : 0) != in->n_matches)
    return fail(LFR_EINVAL, "pair_ptr does not end at n_matches");
  if (in->n_matches && in->n_pairs + 1 > (uint64_t)INT32_MAX) return fail(LFR_EUNSUPPORTED, "2^31 or more listed pairs");
  lfr_options o;
  if (opt) o = *opt; else lfr_options_default(&o);
  LFR_TRY(select_device(o));
  lfr_plan* pl = new lfr_plan();
  pl->device = o.device;
  lfr_host_sizes S;
  MatchArrays d;
  int rc;
  {
    lfr_host_input file_in = *in;  // the decoder sees the file's matches
    file_in.n_matches = src_pair_ptr[n_src_pairs];
    MatchArrays src;
    rc = decode_wire_on_device(&file_in, parts, n_parts, src, 0);
    if (rc == LFR_OK) rc = expand_listed_on_device(src_pair_ptr, n_src_pairs, pair_src, in->n_pairs, in->n_matches, src, d, 0);
  }
  if (rc == LFR_OK) rc = create_plan_from_graph(in, d, o, initial_positions, pl, &S);
  if (rc) {
    free_plan(pl);
    return rc;
  }
  if (sizes) *sizes = S;
  *out = pl;
  return LFR_OK;
}

int lfr_debug_last_wire_times(double* out2) {
  out2[0] = g_wire_ms[0];
  out2[1] = g_wire_ms[1];
  return LFR_OK;
}

int lfr_plan_export_graph(const lfr_plan* pl, uint32_t* row_ptr, lfr_edge* edges, uint32_t* track, uint32_t* comp,
                          uint8_t* is_root, uint32_t* comp_ptr, uint32_t* comp_nodes, uint32_t* comp_order,
                          uint32_t* node_image, uint32_t* node_feat) {
  if (!pl || !pl->graph) return fail(LFR_EINVAL, "plan was not made by lfr_plan_create_from_matches");
  const lfr_plan::GraphArrays& G = *pl->graph;
  auto cp = [](void* dst, const void* src, size_t bytes) {
    if (dst && bytes) std::memcpy(dst, src, bytes);
  };
  cp(row_ptr, G.row_ptr.data(), G.row_ptr.size() * 4);
  cp(track, G.track.data(), G.track.size() * 4);
  cp(comp, G.comp.data(), G.comp.size() * 4);
  cp(is_root, G.is_root.data(), G.is_root.size());
  cp(comp_ptr, G.comp_ptr.data(), G.comp_ptr.size() * 4);
  cp(comp_nodes, G.comp_nodes.data(), G.comp_nodes.size() * 4);
  cp(comp_order, G.comp_order.data(), G.comp_order.size() * 4);
  cp(node_image, G.node_image.data(), G.node_image.size() * 4);
  cp(node_feat, G.node_feat.data(), G.node_feat.size() * 4);
  if (edges && pl->E) {
    LFR_CUDA(cudaSetDevice(pl->device));
    LFR_CUDA(cudaMemcpy(edges, pl->edges.p, sizeof(lfr_edge) * (size_t)pl->E, cudaMemcpyDeviceToHost));
  }
  return LFR_OK;
}

int64_t lfr_plan_encode_solution(lfr_plan* pl, void* stream, uint32_t n_images, const uint8_t* names,
                                 const uint64_t* name_off, const float* fact, uint8_t* out, uint64_t cap,
                                 uint64_t* n_outside) {
  LFR_TRY(check_names(pl, n_images, names, name_off, n_images && (!name_off || !fact) ? "NULL image names or facts" : nullptr));
  LFR_CUDA(cudaSetDevice(pl->device));
  return encode_one(pl, stream, EncodeInput{n_images, names, name_off, fact}, out, cap, n_outside);
}

int64_t lfr_plan_encode_solution_images(lfr_plan* pl, void* stream, uint32_t n_images, const uint8_t* names,
                                        const uint64_t* name_off, const float* fact, const uint8_t* written, uint8_t* out,
                                        uint64_t cap, uint64_t* n_outside) {
  if (!written) return fail(LFR_EINVAL, "written is NULL");
  LFR_TRY(check_names(pl, n_images, names, name_off, n_images && (!name_off || !fact) ? "NULL image names or facts" : nullptr));
  LFR_CUDA(cudaSetDevice(pl->device));
  std::vector<uint32_t> group(n_images);  // one group; an image without the flag is in none
  for (uint32_t k = 0; k < n_images; ++k) group[k] = written[k] ? 0 : 1;
  return encode_one(pl, stream, EncodeInput{n_images, names, name_off, fact, group.data(), 1}, out, cap, n_outside);
}

int64_t lfr_plan_encode_solution_groups(lfr_plan* pl, void* stream, uint32_t n_images, const uint8_t* names,
                                        const uint64_t* name_off, const float* fact, const uint32_t* group_of_image,
                                        uint32_t n_groups, uint8_t* out, uint64_t cap, uint64_t* group_off,
                                        uint64_t* n_outside) {
  const char* missing = n_images && (!name_off || !fact || !group_of_image) ? "NULL image names, facts or groups"
                        : !group_off || (n_groups && !n_outside)           ? "NULL group_off or n_outside"
                                                                           : nullptr;
  LFR_TRY(check_names(pl, n_images, names, name_off, missing, group_of_image, n_groups));
  LFR_CUDA(cudaSetDevice(pl->device));
  std::vector<uint64_t> outside((size_t)n_groups + 1);
  uint64_t carried;
  const int64_t total = encode_solution(pl, (cudaStream_t)stream,
                                        EncodeInput{n_images, names, name_off, fact, group_of_image, n_groups}, out, cap,
                                        group_off, outside.data(), &carried);
  std::copy(outside.begin(), outside.end() - 1, n_outside);
  return total;
}

int lfr_plan_fix_images(lfr_plan* pl, const uint8_t* fixed_by_image_id, uint32_t n_images) {
  if (!pl || !pl->graph) return fail(LFR_EINVAL, "plan was not made by lfr_plan_create_from_matches");
  if (n_images < pl->n_images) return fail(LFR_EINVAL, "n_images is smaller than the plan's image count");
  if (n_images && !fixed_by_image_id) return fail(LFR_EINVAL, "fixed_by_image_id is NULL");
  LFR_CUDA(cudaSetDevice(pl->device));
  pl->fixed_host.assign(fixed_by_image_id, fixed_by_image_id + n_images);
  return build_constant_mask(pl, 0);
}

int lfr_plan_start_from_solution(lfr_plan* pl, void* stream, const uint8_t* bytes, uint64_t len, uint32_t n_images,
                                 const uint8_t* names, const uint64_t* name_off, uint64_t* n_started) {
  lfr::join::Decoded d;
  LFR_TRY(decode_solution_for(pl, bytes, len, n_images, names, name_off, d));
  LFR_CUDA(cudaSetDevice(pl->device));
  return join_solution(pl, (cudaStream_t)stream, d, nullptr, n_started);
}

int lfr_plan_keep_solution(lfr_plan* pl, void* stream, const uint8_t* bytes, uint64_t len, uint32_t n_images,
                           const uint8_t* names, const uint64_t* name_off, uint64_t* n_kept) {
  lfr::join::Decoded d;
  LFR_TRY(decode_solution_for(pl, bytes, len, n_images, names, name_off, d));
  LFR_CUDA(cudaSetDevice(pl->device));
  const cudaStream_t s = (cudaStream_t)stream;
  if (!pl->kept.p) {  // cleared, so that a join that fails before its kernel leaves no stale flags
    LFR_TRY(pl->kept.reserve(std::max<size_t>(pl->N, 1)));
    LFR_CUDA(cudaMemsetAsync(pl->kept.p, 0, std::max<size_t>(pl->N, 1), s));
  }
  LFR_TRY(join_solution(pl, s, d, pl->kept.as<uint8_t>(), n_kept));
  return build_constant_mask(pl, s);
}

int lfr_plan_update_solution(lfr_plan* pl, void* stream, const uint8_t* bytes, uint64_t len, uint32_t n_images,
                             const uint8_t* names, const uint64_t* name_off, uint64_t* n_held, uint32_t* n_touched) {
  lfr::join::Decoded d;
  LFR_TRY(decode_solution_for(pl, bytes, len, n_images, names, name_off, d));
  LFR_CUDA(cudaSetDevice(pl->device));
  return update_solution(pl, (cudaStream_t)stream, d, nullptr, n_held, n_touched);
}

int lfr_plan_update_solution_since(lfr_plan* pl, void* stream, const uint8_t* bytes, uint64_t len, uint32_t n_images,
                                   const uint8_t* names, const uint64_t* name_off, const lfr_plan* previous,
                                   uint32_t prev_n_images, const uint8_t* prev_names, const uint64_t* prev_name_off,
                                   uint64_t* n_held, uint32_t* n_touched, uint32_t* n_changed) {
  lfr::join::Decoded d;
  LFR_TRY(decode_solution_for(pl, bytes, len, n_images, names, name_off, d));
  if (!previous || !previous->graph) return fail(LFR_EINVAL, "previous plan was not made by lfr_plan_create_from_matches");
  if (previous == pl) return fail(LFR_EINVAL, "previous plan is the plan itself");
  if (previous->device != pl->device) return fail(LFR_EINVAL, "previous plan is on another device");
  if (prev_n_images < previous->n_images) return fail(LFR_EINVAL, "prev_n_images is smaller than the previous plan's image count");
  std::vector<uint32_t> image_map;
  if (lfr::join::map_previous_images(n_images, names, name_off, prev_n_images, prev_names, prev_name_off, image_map) != LFR_OK)
    return fail(LFR_EINVAL, "malformed or repeated previous image names");
  LFR_CUDA(cudaSetDevice(pl->device));
  const cudaStream_t s = (cudaStream_t)stream;
  TmpBuf changed;
  LFR_TRY(changed.reserve(std::max<size_t>(pl->C, 1)));
  uint32_t nc = 0;
  LFR_TRY(diff_components(pl, previous, image_map, s, changed.as<uint8_t>(), &nc));
  LFR_TRY(update_solution(pl, s, d, changed.as<uint8_t>(), n_held, n_touched));
  if (n_changed) *n_changed = nc;
  return LFR_OK;
}

int64_t lfr_plan_problem_record(lfr_plan* pl, void* stream, uint32_t n_images, const uint8_t* names,
                                const uint64_t* name_off, uint8_t* out, uint64_t cap) {
  LFR_TRY(check_names(pl, n_images, names, name_off, n_images && !name_off ? "NULL image names" : nullptr));
  const uint32_t C = pl->C;
  const uint64_t need = lfr::record::record_bytes(C);
  if (!out || cap < need) return (int64_t)need;
  LFR_CUDA(cudaSetDevice(pl->device));
  const cudaStream_t s = (cudaStream_t)stream;
  TmpBuf d0, d1, k1, v0, tmp;
  LFR_TRY(plan_digests(pl, s, n_images, names, name_off, d0, d1));
  std::vector<unsigned long long> h0(C), h1(C);
  if (C) {
    LFR_TRY(k1.reserve(8 * (size_t)C));
    LFR_TRY(v0.reserve(8 * (size_t)C));
    auto* a0 = d0.as<unsigned long long>();
    auto* a1 = d1.as<unsigned long long>();
    auto* b1 = k1.as<unsigned long long>();
    auto* b0 = v0.as<unsigned long long>();
    // ascending (d0, d1): by d1, then stably by d0
    LFR_TRY(cub_run(tmp, [&](void* t, size_t& nb) { return cub::DeviceRadixSort::SortPairs(t, nb, a1, b1, a0, b0, (int)C, 0, 64, s); }));
    LFR_TRY(cub_run(tmp, [&](void* t, size_t& nb) { return cub::DeviceRadixSort::SortPairs(t, nb, b0, a0, b1, a1, (int)C, 0, 64, s); }));
    LFR_CUDA(cudaMemcpyAsync(h0.data(), a0, 8 * (size_t)C, cudaMemcpyDeviceToHost, s));
    LFR_TRY(fetch(h1.data(), a1, C, s));
  }
  lfr::record::store_u64(out, lfr::record::kMagic);
  lfr::record::store_u64(out + 8, C);
  for (uint32_t c = 0; c < C; ++c) {
    lfr::record::store_u64(out + lfr::record::kHeaderBytes + 16 * (size_t)c, h0[c]);
    lfr::record::store_u64(out + lfr::record::kHeaderBytes + 16 * (size_t)c + 8, h1[c]);
  }
  return (int64_t)need;
}

int lfr_plan_update_solution_since_record(lfr_plan* pl, void* stream, const uint8_t* bytes, uint64_t len, uint32_t n_images,
                                          const uint8_t* names, const uint64_t* name_off, const uint8_t* record,
                                          uint64_t record_len, uint64_t* n_held, uint32_t* n_touched, uint32_t* n_changed) {
  lfr::join::Decoded d;
  LFR_TRY(decode_solution_for(pl, bytes, len, n_images, names, name_off, d));
  LFR_TRY(check_names(pl, n_images, names, name_off, n_images && !name_off ? "NULL image names" : nullptr));
  uint64_t R = 0;
  if (!lfr::record::check(record, record_len, &R)) return fail(LFR_EINVAL, "malformed problem record");
  LFR_CUDA(cudaSetDevice(pl->device));
  const cudaStream_t s = (cudaStream_t)stream;
  const uint32_t C = pl->C;
  TmpBuf d0, d1, d_rec, changed, d_ctr;
  LFR_TRY(plan_digests(pl, s, n_images, names, name_off, d0, d1));
  LFR_TRY(changed.reserve(std::max<size_t>(C, 1)));
  LFR_TRY(d_rec.reserve(std::max<uint64_t>(16 * R, 16)));
  LFR_TRY(d_ctr.reserve(8));
  LFR_CUDA(cudaMemsetAsync(changed.p, 0, std::max<size_t>(C, 1), s));
  LFR_CUDA(cudaMemsetAsync(d_ctr.p, 0, 8, s));
  unsigned long long nc = 0;
  if (C) {
    if (R) LFR_CUDA(cudaMemcpyAsync(d_rec.p, record + lfr::record::kHeaderBytes, 16 * R, cudaMemcpyHostToDevice, s));
    lfr::record::lookup_kernel<<<blocks_for(C), 256, 0, s>>>(d0.as<unsigned long long>(), d1.as<unsigned long long>(), C,
                                                             d_rec.as<ulonglong2>(), R, changed.as<uint8_t>());
    lfr::start::count_touched_kernel<<<blocks_for(C), 256, 0, s>>>(changed.as<uint8_t>(), C, d_ctr.as<unsigned long long>());
    LFR_LAUNCHED();
    LFR_TRY(fetch(&nc, d_ctr.p, 1, s));  // also orders the record's upload before the caller's buffer may go
  }
  LFR_TRY(update_solution(pl, s, d, changed.as<uint8_t>(), n_held, n_touched));
  if (n_changed) *n_changed = (uint32_t)nc;
  return LFR_OK;
}

int lfr_plan_update_solution_groups(lfr_plan* pl, void* stream, uint32_t n_images, const uint8_t* names,
                                    const uint64_t* name_off, const uint32_t* group_of_image, uint32_t n_groups,
                                    const uint8_t* const* files, const uint64_t* file_len, const uint8_t* const* records,
                                    const uint64_t* record_len, uint64_t* n_held, uint32_t* n_touched, uint32_t* n_changed) {
  const uint32_t G = n_groups;
  const char* missing = n_images && (!name_off || !group_of_image)                        ? "NULL image names or groups"
                        : G && ((files && !file_len) || (records && !record_len))           ? "NULL file_len or record_len"
                                                                                            : nullptr;
  LFR_TRY(check_names(pl, n_images, names, name_off, missing, group_of_image, G));
  // every record checked, and every scene's digests back to back: scene g's in [rec_off[g], rec_off[g + 1])
  std::vector<uint64_t> rec_off((size_t)G + 1, 0);
  std::vector<uint8_t> has_rec(std::max<uint32_t>(G, 1), 0), rec_bytes;
  for (uint32_t g = 0; g < G; ++g) {
    uint64_t R = 0;
    if (records && records[g]) {
      if (!lfr::record::check(records[g], record_len[g], &R)) return fail(LFR_EINVAL, "malformed problem record");
      has_rec[g] = 1;
      rec_bytes.insert(rec_bytes.end(), records[g] + lfr::record::kHeaderBytes, records[g] + record_len[g]);
    }
    rec_off[g + 1] = rec_off[g] + R;
  }
  const bool any_rec = std::find(has_rec.begin(), has_rec.end(), (uint8_t)1) != has_rec.end();
  lfr::join::Decoded d;
  const uint8_t no_name = 0;
  if (lfr::join::decode_groups(G, files, file_len, n_images, names ? names : &no_name, name_off, group_of_image, d) != LFR_OK)
    return fail(LFR_EINVAL, "malformed SolutionFile");
  if (d.n_disp >= (1ull << 31)) return fail(LFR_EUNSUPPORTED, "SolutionFiles with 2^31 or more displacements");
  LFR_CUDA(cudaSetDevice(pl->device));
  const cudaStream_t s = (cudaStream_t)stream;
  const uint32_t C = pl->C;
  TmpBuf d0, d1, d_group, cgroup, d_rec, d_rec_off, d_has, changed, d_ctr;
  unsigned long long nc = 0;
  if (any_rec && C) {
    // the digests, each component's scene, and one lookup of every component in its own scene's record
    LFR_TRY(plan_digests(pl, s, n_images, names, name_off, d0, d1));
    LFR_TRY(component_groups(pl, s, n_images, group_of_image, d_group, cgroup));
    LFR_TRY(upload(&d_rec, rec_bytes.data(), rec_bytes.size(), s));
    LFR_TRY(upload(&d_rec_off, rec_off.data(), rec_off.size(), s));
    LFR_TRY(upload(&d_has, has_rec.data(), has_rec.size(), s));
    LFR_TRY(changed.reserve(C));
    LFR_TRY(d_ctr.reserve(8));
    LFR_CUDA(cudaMemsetAsync(d_ctr.p, 0, 8, s));
    lfr::record::group_lookup_kernel<<<blocks_for(C), 256, 0, s>>>(
        d0.as<unsigned long long>(), d1.as<unsigned long long>(), cgroup.as<uint32_t>(), C, d_rec.as<ulonglong2>(),
        d_rec_off.as<uint64_t>(), d_has.as<uint8_t>(), changed.as<uint8_t>());
    lfr::start::count_touched_kernel<<<blocks_for(C), 256, 0, s>>>(changed.as<uint8_t>(), C, d_ctr.as<unsigned long long>());
    LFR_LAUNCHED();
    LFR_TRY(fetch(&nc, d_ctr.p, 1, s));  // also orders the uploads before the host vectors go
  }
  LFR_TRY(update_solution(pl, s, d, any_rec && C ? changed.as<uint8_t>() : nullptr, n_held, n_touched));
  if (n_changed) *n_changed = (uint32_t)nc;
  return LFR_OK;
}

int64_t lfr_plan_problem_record_groups(lfr_plan* pl, void* stream, uint32_t n_images, const uint8_t* names,
                                       const uint64_t* name_off, const uint32_t* group_of_image, uint32_t n_groups,
                                       uint8_t* out, uint64_t cap, uint64_t* group_off) {
  const uint32_t G = n_groups;
  const char* missing = n_images && (!name_off || !group_of_image) ? "NULL image names or groups"
                        : !group_off                                 ? "NULL group_off"
                                                                     : nullptr;
  LFR_TRY(check_names(pl, n_images, names, name_off, missing, group_of_image, G));
  LFR_CUDA(cudaSetDevice(pl->device));
  const cudaStream_t s = (cudaStream_t)stream;
  const uint32_t C = pl->C;
  TmpBuf d0, d1, d_group, cgroup, iota, k1, i1, k0, k0s, i2, kg, kgs, i3, goff, tmp;
  // the digests and each component's scene; then (group, d0, d1) order by three stable radix sorts of an index:
  // by d1, by d0, by group
  LFR_TRY(plan_digests(pl, s, n_images, names, name_off, d0, d1));
  LFR_TRY(component_groups(pl, s, n_images, group_of_image, d_group, cgroup));
  for (TmpBuf* b : {&iota, &i1, &i2, &kg, &kgs, &i3}) LFR_TRY(b->reserve(4 * std::max<size_t>(C, 1)));
  for (TmpBuf* b : {&k1, &k0, &k0s}) LFR_TRY(b->reserve(8 * std::max<size_t>(C, 1)));
  LFR_TRY(goff.reserve(8 * ((size_t)G + 1)));
  const auto* a0 = d0.as<unsigned long long>();
  const auto* a1 = d1.as<unsigned long long>();
  if (C) {
    lfr::graph::iota_kernel<<<blocks_for(C), 256, 0, s>>>(iota.as<uint32_t>(), C);
    LFR_LAUNCHED();
    LFR_TRY(cub_run(tmp, [&](void* t, size_t& nb) {
      return cub::DeviceRadixSort::SortPairs(t, nb, a1, k1.as<unsigned long long>(), iota.as<uint32_t>(), i1.as<uint32_t>(),
                                             (int)C, 0, 64, s);
    }));
    lfr::record::gather_u64_kernel<<<blocks_for(C), 256, 0, s>>>(a0, i1.as<uint32_t>(), C, k0.as<unsigned long long>());
    LFR_LAUNCHED();
    LFR_TRY(cub_run(tmp, [&](void* t, size_t& nb) {
      return cub::DeviceRadixSort::SortPairs(t, nb, k0.as<unsigned long long>(), k0s.as<unsigned long long>(), i1.as<uint32_t>(),
                                             i2.as<uint32_t>(), (int)C, 0, 64, s);
    }));
    lfr::record::gather_u32_kernel<<<blocks_for(C), 256, 0, s>>>(cgroup.as<uint32_t>(), i2.as<uint32_t>(), C, kg.as<uint32_t>());
    LFR_LAUNCHED();
    LFR_TRY(cub_run(tmp, [&](void* t, size_t& nb) {
      return cub::DeviceRadixSort::SortPairs(t, nb, kg.as<uint32_t>(), kgs.as<uint32_t>(), i2.as<uint32_t>(), i3.as<uint32_t>(),
                                             (int)C, 0, bits_for(G), s);
    }));
  }
  lfr::record::record_group_off_kernel<<<blocks_for((uint64_t)G + 1), 256, 0, s>>>(kgs.as<uint32_t>(), C, G, goff.as<uint64_t>());
  LFR_LAUNCHED();
  LFR_TRY(fetch(group_off, goff.p, (size_t)G + 1, s));
  const uint64_t total = group_off[G];
  if (!out || cap < total || !total) return (int64_t)total;
  LFR_TRY(pl->enc_out.reserve(total));
  lfr::record::record_write_kernel<<<blocks_for((uint64_t)C + G), 256, 0, s>>>(a0, a1, i3.as<uint32_t>(), kgs.as<uint32_t>(), C, G,
                                                                                goff.as<uint64_t>(), pl->enc_out.as<uint8_t>());
  LFR_LAUNCHED();
  LFR_TRY(fetch(out, pl->enc_out.p, total, s));
  return (int64_t)total;
}

int lfr_debug_device_ops(unsigned long long* out3, int reset) {
  for (int k = 0; k < 3; ++k) {
    if (out3) out3[k] = g_device_ops[k];
    if (reset) g_device_ops[k] = 0;
  }
  return LFR_OK;
}

int64_t lfr_plan_encode_solution_carried(lfr_plan* pl, void* stream, uint32_t n_images, const uint8_t* names,
                                         const uint64_t* name_off, const float* fact, const uint8_t* file,
                                         uint64_t file_len, uint8_t* out, uint64_t cap, uint64_t* n_outside,
                                         uint64_t* n_carried) {
  lfr::join::Decoded d;
  LFR_TRY(decode_solution_for(pl, file, file_len, n_images, names, name_off, d));
  if (n_images && !fact) return fail(LFR_EINVAL, "NULL image facts");
  {
    const char* nm = names ? reinterpret_cast<const char*>(names) : "";
    std::unordered_set<std::string> seen;
    seen.reserve(n_images);
    for (uint32_t k = 0; k < n_images; ++k)
      if (!seen.emplace(nm + name_off[k], name_off[k + 1] - name_off[k]).second)
        return fail(LFR_EINVAL, "repeated image name");
  }
  if ((uint64_t)pl->N + d.n_disp >= (1ull << 31)) return fail(LFR_EUNSUPPORTED, "2^31 or more nodes and displacements");
  LFR_CUDA(cudaSetDevice(pl->device));
  return encode_one(pl, stream, EncodeInput{n_images, names, name_off, fact, nullptr, 1, file, &d}, out, cap, n_outside,
                    n_carried);
}

int lfr_debug_last_encode_times(double* out2) {
  out2[0] = g_encode_ms[0];
  out2[1] = g_encode_ms[1];
  return LFR_OK;
}

int lfr_graph_stage_on_device(const lfr_host_input* in, int32_t n_devices) {
  // host code only: decided before any CUDA call, so a one-shot process can choose its route while the
  // context is still being created
  if (!in || n_devices != 1) return 0;
  if (in->n_images > 65535 || in->n_pairs + 1 >= (1ull << 31)) return 0;  // the device stage refuses these
  if (in->n_pairs && (!in->pair_ptr || in->pair_ptr[in->n_pairs] > in->n_matches)) return 0;
  uint64_t e = 0;
  for (uint64_t p = 0; p < in->n_pairs; ++p) {
    if (in->pair_ptr[p + 1] < in->pair_ptr[p]) return 0;  // malformed: the host stage reports it
    if (!(in->pair_skip && in->pair_skip[p])) e += 2 * (in->pair_ptr[p + 1] - in->pair_ptr[p]);
  }
  return e >= kDeviceGraphStageMinEdges && e < (1ull << 31) ? 1 : 0;
}

int lfr_wire_decode_on_device(uint64_t n_matches) { return n_matches >= kDeviceDecodeMinMatches ? 1 : 0; }

int lfr_plan_solve(lfr_plan* pl, void* stream) {
  if (!pl) return fail(LFR_EINVAL, "plan is NULL");
  LFR_CUDA(cudaSetDevice(pl->device));
  return launch_solve(pl, (cudaStream_t)stream);
}

int lfr_plan_num_launches(const lfr_plan* pl) {
  // kernels only: the device-to-device reset of `positions` is a copy, not a kernel
  return pl ? pl->num_launches() : 0;
}

int lfr_plan_download(lfr_plan* pl, void* stream, double* positions, lfr_stats* st) {
  if (!pl) return fail(LFR_EINVAL, "plan is NULL");
  LFR_CUDA(cudaSetDevice(pl->device));
  return download(pl, (cudaStream_t)stream, positions, st);
}

int lfr_plan_traffic(lfr_plan* pl, void* stream, uint64_t* algorithmic_bytes, uint64_t* one_pass_bytes) {
  if (!pl) return fail(LFR_EINVAL, "plan is NULL");
  LFR_CUDA(cudaSetDevice(pl->device));
  cudaStream_t s = (cudaStream_t)stream;
  std::vector<unsigned char> blk(pl->stats_bytes());
  LFR_CUDA(cudaMemcpyAsync(blk.data(), pl->stats.p, blk.size(), cudaMemcpyDeviceToHost, s));
  LFR_CUDA(cudaStreamSynchronize(s));
  const int32_t* it = reinterpret_cast<const int32_t*>(blk.data() + 16 * (size_t)pl->Cp);
  const uint32_t* kept = reinterpret_cast<const uint32_t*>(blk.data() + 16 * (size_t)pl->Cp + 12 * (size_t)pl->Cp);
  uint64_t alg = 0, one = 0;
  for (uint32_t c = 0; c < pl->C; ++c) {
    if (pl->comp_size[c] <= 1) continue;
    const uint64_t pass = 80ull * kept[c] + 36ull * pl->comp_size[c];  // SURVEY 8d
    one += pass;
    alg += pass * (uint64_t)std::max(it[c], 1);
  }
  if (algorithmic_bytes) *algorithmic_bytes = alg;
  if (one_pass_bytes) *one_pass_bytes = one;
  return LFR_OK;
}

/* debug (LFR_DBG_PROFILE): one lfr::LmProfile record per slot, 8 x uint64 each:
   0 total cycles, 1 setup, 2 evaluation, 3 assembly, 4 linear solve, 5 line search and the rest,
   6 line-search steps << 32 | SM id, 7 tier << 56 | tier counter (see lfr_lm.cuh) */
int lfr_debug_plan_cycles(lfr_plan* pl, unsigned long long* out) {
  if (!pl || !pl->profile) return fail(LFR_EINVAL, "plan was not created with LFR_DBG_PROFILE");
  LFR_CUDA(cudaSetDevice(pl->device));
  LFR_CUDA(cudaMemcpy(out, pl->cycles.p, sizeof(unsigned long long) * 8 * (size_t)pl->C, cudaMemcpyDeviceToHost));
  return LFR_OK;
}

int lfr_debug_plan_times(lfr_plan* pl, unsigned long long* out) {
  if (!pl || !pl->profile) return fail(LFR_EINVAL, "plan was not created with LFR_DBG_PROFILE");
  LFR_CUDA(cudaSetDevice(pl->device));
  LFR_CUDA(cudaMemcpy(out, pl->times.p, sizeof(unsigned long long) * 2 * (size_t)pl->C, cudaMemcpyDeviceToHost));
  return LFR_OK;
}

/* debug (LFR_DBG_PROFILE): counters of the last lfr_solve() of this thread on `device`:
   cycles [8 per slot], times [2 per slot] = %globaltimer ns at start / end of each component */
int lfr_debug_last_solve_profile(int device, unsigned long long* cycles, unsigned long long* times) {
  if (device < 0 || device >= kMaxDevices || !g_ws[device].ready || !g_ws[device].plan->profile)
    return fail(LFR_EINVAL, "no profiled lfr_solve() on this device / thread");
  lfr_plan* pl = g_ws[device].plan;
  LFR_CUDA(cudaSetDevice(device));
  if (cycles) LFR_CUDA(cudaMemcpy(cycles, pl->cycles.p, sizeof(unsigned long long) * 8 * (size_t)pl->C, cudaMemcpyDeviceToHost));
  if (times) LFR_CUDA(cudaMemcpy(times, pl->times.p, sizeof(unsigned long long) * 2 * (size_t)pl->C, cudaMemcpyDeviceToHost));
  return LFR_OK;
}

// host-only: best-of-`reps` time of the schedule construction (build_schedule), no device needed
int lfr_debug_time_schedule(const lfr_problem* p, const lfr_options* opt, int reps, double* best_us, int* n_launches,
                            uint64_t* digest) {
  if (!p || !best_us) return fail(LFR_EINVAL, "null argument");
  LFR_TRY(validate(p));
  lfr_plan pl;
  if (opt) pl.opt = *opt; else lfr_options_default(&pl.opt);
  pl.N = p->n_nodes;
  pl.C = p->n_components;
  pl.total_slots = p->n_components ? p->comp_ptr[p->n_components] : 0;
  double best = 1e300;
  for (int r = 0; r < std::max(reps, 1); ++r) {
    const auto t0 = std::chrono::steady_clock::now();
    LFR_TRY(build_schedule(&pl, p));
    best = std::min(best, std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now() - t0).count());
  }
  if (std::getenv("LFR_SCHED_DUMP")) {  // the bucket launches, the queue launches, then the CTA tier
    for (const Launch& L : pl.launches)
      if (L.kernel != Kernel::kQueue && !is_cta(L.kernel))
        std::fprintf(stderr, "bucket variant %3d  n %6u  emax %5d ncmax %4d n2max %3d  smem/warp %6d  warps %d  -> CTAs/SM by smem %d\n",
                     info(L.kernel).label, L.n, L.emax, L.ncmax, L.n2max, L.bytes, L.warps,
                     (int)(kMaxSmemPerBlock / (L.bytes * L.warps + 1024)));
    for (const Launch& L : pl.launches)
      if (L.kernel == Kernel::kQueue) std::fprintf(stderr, "warp2 queue  n %6u  slot %6d  warps/SM %d\n", L.n, L.bytes, L.warps);
    std::fprintf(stderr, "CTA tier: %zu components\n", pl.large_slots.size());
    for (const Launch& L : pl.launches)
      if (is_cta(L.kernel))
        std::fprintf(stderr, "cta group  n %6u  max_free %6u  minb %d  smem_vecs %d  smem %6d\n", L.n, L.max_free,
                     info(L.kernel).label, L.smem_vecs, L.bytes);
  }
  if (digest) {  // FNV-1a over everything the launches depend on: the schedule must not depend on the thread count
    uint64_t h = 1469598103934665603ull;
    auto mix = [&](uint64_t v) {
      for (int i = 0; i < 8; ++i) {
        h ^= (v >> (8 * i)) & 0xff;
        h *= 1099511628211ull;
      }
    };
    mix(pl.n_solved);
    for (const Launch& L : pl.launches) {
      mix((uint64_t)L.kernel); mix(L.offset); mix(L.n); mix((uint64_t)L.emax); mix((uint64_t)L.ncmax);
      mix((uint64_t)L.n2max); mix((uint64_t)L.bytes); mix((uint64_t)L.warps); mix(L.max_free); mix((uint64_t)L.smem_vecs);
    }
    for (uint32_t c : pl.list_host) mix(c);
    for (size_t i = 0; i < pl.large_slots.size(); ++i) {
      mix(pl.large_slots[i]); mix(pl.large_cand[i]); mix(pl.large_free[i]); mix(pl.large_ell[i]);
    }
    *digest = h;
  }
  *best_us = best;
  if (n_launches) *n_launches = pl.num_launches();
  return LFR_OK;
}

int lfr_debug_last_host_marks(double* out6) {
  for (int i = 0; i < 6; ++i) out6[i] = g_host_marks[i];
  return LFR_OK;
}

#ifdef LFR_POLY_PROF
/* diagnostic build only: cycle split of the line-search polynomial (lfr_math.cuh) */
int lfr_debug_poly_prof(unsigned long long* out16, int reset) {
  LFR_CUDA(cudaMemcpyFromSymbol(out16, lfr::g_poly_prof, sizeof(unsigned long long) * 16));
  if (reset) {
    unsigned long long z[16] = {0};
    LFR_CUDA(cudaMemcpyToSymbol(lfr::g_poly_prof, z, sizeof(z)));
  }
  return LFR_OK;
}
#endif

void lfr_plan_destroy(lfr_plan* pl) {
  if (!pl) return;
  cudaSetDevice(pl->device);
  free_plan(pl);
}

int lfr_solve(const lfr_problem* p, const lfr_options* opt, double* positions, lfr_stats* st) {
  LFR_TRY(validate(p));
  if (p->n_nodes && !positions) return fail(LFR_EINVAL, "positions is NULL");
  lfr_options o;
  if (opt) o = *opt; else lfr_options_default(&o);
  if (o.device < 0 || o.device >= kMaxDevices) return fail(LFR_EUNSUPPORTED, "device ordinal out of [0, 16)");
  std::lock_guard<std::mutex> lock(g_ws_mutex[o.device]);
  // One device: the copy engine moves the edge records to HBM at full link rate; the kernels' own
  // pulls over PCIe take more than twice as long end to end on an H100 (DESIGN.md §4): opt-in here.
  return solve_on_device(p, o, positions, st, nullptr, 0, nullptr, (o.debug_flags & LFR_DBG_ZERO_COPY) != 0);
}

void* lfr_host_alloc(uint64_t bytes) {
  void* p = nullptr;
  if (cudaHostAlloc(&p, bytes ? (size_t)bytes : 1, cudaHostAllocPortable) != cudaSuccess) {
    cudaGetLastError();
    return nullptr;
  }
  return p;
}

void lfr_host_free(void* p) {
  if (p) cudaFreeHost(p);
}

void lfr_shutdown(void) {
  // release the cached per-device workspaces of lfr_solve() / lfr_solve_multi() (device buffers,
  // pinned staging, streams, events); the next call re-creates what it needs
  for (int d = 0; d < kMaxDevices; ++d) {
    std::lock_guard<std::mutex> lock(g_ws_mutex[d]);
    DeviceWorkspace& ws = g_ws[d];
    if (!ws.ready) continue;
    if (cudaSetDevice(d) == cudaSuccess) {
      free_plan(ws.plan);
      for (int i = 0; i < 4; ++i)
        if (ws.ev[i]) cudaEventDestroy(ws.ev[i]);
      if (ws.stream) cudaStreamDestroy(ws.stream);
    }
    ws = DeviceWorkspace();
  }
}

int lfr_solve_multi(const lfr_problem* p, const lfr_options* opt, const int32_t* devices, int32_t n_devices,
                    double* positions, lfr_stats* st, lfr_multi_info* info) {
  LFR_TRY(validate(p));
  if (p->n_nodes && !positions) return fail(LFR_EINVAL, "positions is NULL");
  if (!devices || n_devices < 1 || n_devices > kMaxDevices) return fail(LFR_EINVAL, "devices: need 1..16 device ordinals");
  for (int d = 0; d < n_devices; ++d) {
    if (devices[d] < 0 || devices[d] >= kMaxDevices) return fail(LFR_EUNSUPPORTED, "device ordinal out of [0, 16)");
    for (int e = 0; e < d; ++e)
      if (devices[e] == devices[d]) return fail(LFR_EINVAL, "devices: duplicate ordinal");
  }
  lfr_options o0;
  if (opt) o0 = *opt; else lfr_options_default(&o0);
  const uint32_t C = p->n_components;
  // ---- LPT packing of the dispatch slots by directed-edge count, largest first (the reference's
  // largest-first queue, solve.cc:599-604, spread over devices); deterministic
  std::vector<uint64_t> weight(C, 0);
  const uint32_t total_slots = C ? p->comp_ptr[C] : 0;
  for (uint32_t c = 0; c < C; ++c) {
    const uint32_t beg = p->comp_ptr[c], end = p->comp_ptr[c + 1];
    if (end < beg || end > total_slots) return fail(LFR_EINVAL, "comp_ptr not monotone");
    if (end - beg <= 1) continue;
    for (uint32_t i = beg; i < end; ++i) {
      const uint32_t v = p->comp_nodes[i];
      if (v >= p->n_nodes) return fail(LFR_EINVAL, "comp_nodes out of range");
      weight[c] += p->row_ptr[v + 1] - p->row_ptr[v];
    }
  }
  std::vector<uint32_t> order(C);
  for (uint32_t c = 0; c < C; ++c) order[c] = c;
  std::stable_sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return weight[a] > weight[b]; });
  std::vector<uint8_t> owner(C, 0);
  std::vector<uint64_t> load(n_devices, 0);
  std::vector<uint32_t> n_slots(n_devices, 0);
  for (uint32_t c : order) {
    int best = 0;
    for (int d = 1; d < n_devices; ++d)
      if (load[d] < load[best]) best = d;
    owner[c] = (uint8_t)best;
    load[best] += weight[c];
    if (weight[c]) ++n_slots[best];
  }
  // ---- one host thread per device: upload the (small) per-node arrays, launch, collect.  With
  // page-locked caller buffers every device pulls only ITS components' edge records from the shared
  // host array and writes its results straight into `positions` (disjoint entries): the edge data is
  // partitioned without ever being copied, and no collective is needed.
  std::vector<lfr_stats> dst(n_devices);
  std::vector<std::vector<int32_t>> d_iter(n_devices), d_term(n_devices);
  std::vector<std::vector<double>> d_c0(n_devices), d_c1(n_devices), d_pos(n_devices);
  std::vector<int> rcs(n_devices, LFR_OK);
  std::vector<std::string> errs(n_devices);
  const bool pos_pinned = !(o0.debug_flags & LFR_DBG_NO_ZERO_COPY) && p->n_nodes && device_view_of_pinned(positions) != nullptr;
  auto work = [&](int d) {
    lfr_options o = o0;
    o.device = devices[d];
    std::memset(&dst[d], 0, sizeof(lfr_stats));
    d_iter[d].assign(C, 0);
    d_term[d].assign(C, 0);
    d_c0[d].assign(C, 0.0);
    d_c1[d].assign(C, 0.0);
    dst[d].iterations = d_iter[d].data();
    dst[d].termination = d_term[d].data();
    dst[d].initial_cost = d_c0[d].data();
    dst[d].final_cost = d_c1[d].data();
    if (!pos_pinned) d_pos[d].assign(2 * (size_t)p->n_nodes, 0.0);
    std::lock_guard<std::mutex> lock(g_ws_mutex[o.device]);
    rcs[d] = solve_on_device(p, o, positions, &dst[d], owner.data(), (uint8_t)d, pos_pinned ? nullptr : d_pos[d].data(),
                            /*in_place=*/true);
    if (rcs[d]) errs[d] = g_last_error;
  };
  if (n_devices == 1) {
    work(0);
  } else {
    std::vector<std::thread> threads;
    for (int d = 0; d < n_devices; ++d) threads.emplace_back(work, d);
    for (auto& t : threads) t.join();
  }
  for (int d = 0; d < n_devices; ++d)
    if (rcs[d]) return fail(rcs[d], "device " + std::to_string(devices[d]) + ": " + errs[d]);
  // ---- merge by owner
  if (!pos_pinned) {
    for (uint32_t c = 0; c < C; ++c) {
      const uint32_t beg = p->comp_ptr[c], end = p->comp_ptr[c + 1];
      if (end - beg <= 1) continue;
      const double* src = d_pos[owner[c]].data();
      for (uint32_t i = beg; i < end; ++i) {
        const size_t v = p->comp_nodes[i];
        positions[2 * v] = src[2 * v];
        positions[2 * v + 1] = src[2 * v + 1];
      }
    }
  }
  if (st) {
    uint64_t ti = 0, tl = 0;
    uint32_t ns = 0, nk = 0;
    double h = 0, k = 0, dd = 0, tt = 0;
    for (int d = 0; d < n_devices; ++d) {
      ti += dst[d].total_iterations;
      tl += dst[d].total_line_search_steps;
      ns += dst[d].n_solved;
      nk += dst[d].n_kernel_launches;
      h = std::max(h, dst[d].h2d_ms);
      k = std::max(k, dst[d].kernel_ms);
      dd = std::max(dd, dst[d].d2h_ms);
      tt = std::max(tt, dst[d].total_ms);
    }
    for (uint32_t c = 0; c < C; ++c) {
      const int d = owner[c];
      if (st->iterations) st->iterations[c] = d_iter[d][c];
      if (st->termination) st->termination[c] = d_term[d][c];
      if (st->initial_cost) st->initial_cost[c] = d_c0[d][c];
      if (st->final_cost) st->final_cost[c] = d_c1[d][c];
    }
    st->total_iterations = ti;
    st->total_line_search_steps = tl;
    st->n_solved = ns;
    st->n_kernel_launches = nk;
    st->h2d_ms = h;       // maxima over the devices (they run concurrently)
    st->kernel_ms = k;
    st->d2h_ms = dd;
    st->total_ms = tt;
  }
  if (info) {
    for (int d = 0; d < n_devices && d < 16; ++d) {
      info->kernel_ms[d] = dst[d].kernel_ms;
      info->total_ms[d] = dst[d].total_ms;
      info->n_slots[d] = n_slots[d];
      info->n_edges[d] = load[d];
    }
    info->zero_copy = (pos_pinned && p->n_edges && device_view_of_pinned(p->edges) != nullptr) ? 1 : 0;
  }
  return LFR_OK;
}

int lfr_debug_edge_eval(const lfr_edge* edges, const uint8_t* kind, uint64_t n, const double* xs,
                        const double* xd, const lfr_options* opt, double* r, double* jac, double* rho) {
  lfr_options o;
  if (opt) o = *opt; else lfr_options_default(&o);
  LFR_TRY(select_device(o));
  if (n == 0) return LFR_OK;
  DevBuf d_e, d_k, d_xs, d_xd, d_r, d_j, d_rho;
  int rc = LFR_OK;
  auto run = [&]() -> int {
    LFR_TRY(upload(&d_e, edges, n, 0));
    LFR_TRY(upload(&d_k, kind, n, 0));
    LFR_TRY(upload(&d_xs, xs, 2 * n, 0));
    LFR_TRY(upload(&d_xd, xd, 2 * n, 0));
    LFR_TRY(d_r.reserve(n * 16));
    LFR_TRY(d_j.reserve(n * 32));
    LFR_TRY(d_rho.reserve(n * 24));
    lfr::edge_eval_kernel<<<(unsigned)((n + 127) / 128), 128>>>(d_e.as<float4>(), d_k.as<uint8_t>(), n,
                                                               d_xs.as<double>(), d_xd.as<double>(),
                                                               make_consts(o), d_r.as<double>(), d_j.as<double>(),
                                                               d_rho.as<double>());
    LFR_CUDA(cudaGetLastError());
    LFR_CUDA(cudaMemcpy(r, d_r.p, n * 16, cudaMemcpyDeviceToHost));
    LFR_CUDA(cudaMemcpy(jac, d_j.p, n * 32, cudaMemcpyDeviceToHost));
    LFR_CUDA(cudaMemcpy(rho, d_rho.p, n * 24, cudaMemcpyDeviceToHost));
    return LFR_OK;
  };
  rc = run();
  d_e.release(); d_k.release(); d_xs.release(); d_xd.release(); d_r.release(); d_j.release(); d_rho.release();
  return rc;
}

/* test hook: real roots in [lo, hi] of n quartics (5 coefficients each, highest degree first,
   leading coefficient != 0) by the line search's root finders; use_grid = 1 -> Budan-Fourier grid
   isolation (the production route), 0 -> derivative recursion */
int lfr_debug_quartic_roots(const double* coef, const double* lohi, uint64_t n, int use_grid, double* roots,
                            int* counts) {
  lfr_options o;
  lfr_options_default(&o);
  LFR_TRY(select_device(o));
  if (n == 0) return LFR_OK;
  DevBuf d_c, d_l, d_r, d_n;
  auto run = [&]() -> int {
    LFR_TRY(upload(&d_c, coef, 5 * n, 0));
    LFR_TRY(upload(&d_l, lohi, 2 * n, 0));
    LFR_TRY(d_r.reserve(n * 32));
    LFR_TRY(d_n.reserve(n * 4));
    lfr::quartic_roots_kernel<<<(unsigned)((n + 3) / 4), 128>>>(d_c.as<double>(), d_l.as<double>(), (int)n, use_grid,
                                                                d_r.as<double>(), d_n.as<int>());
    LFR_CUDA(cudaGetLastError());
    LFR_CUDA(cudaMemcpy(roots, d_r.p, n * 32, cudaMemcpyDeviceToHost));
    LFR_CUDA(cudaMemcpy(counts, d_n.p, n * 4, cudaMemcpyDeviceToHost));
    return LFR_OK;
  };
  const int rc = run();
  d_c.release(); d_l.release(); d_r.release(); d_n.release();
  return rc;
}

/* test hook: the line search's interpolating-polynomial minimiser on n cases of 11 doubles
   {f0, g0, x1, f1, g1, three, x2, f2, g2, lo, hi}; out[n] = selected step size */
int lfr_debug_ls_minimizer(const double* cases, uint64_t n, double* out) {
  lfr_options o;
  lfr_options_default(&o);
  LFR_TRY(select_device(o));
  if (n == 0) return LFR_OK;
  DevBuf d_i, d_o;
  auto run = [&]() -> int {
    LFR_TRY(upload(&d_i, cases, 11 * n, 0));
    LFR_TRY(d_o.reserve(n * 8));
    lfr::ls_minimizer_kernel<<<(unsigned)((n + 3) / 4), 128>>>(d_i.as<double>(), (int)n, d_o.as<double>());
    LFR_CUDA(cudaGetLastError());
    LFR_CUDA(cudaMemcpy(out, d_o.p, n * 8, cudaMemcpyDeviceToHost));
    return LFR_OK;
  };
  const int rc = run();
  d_i.release(); d_o.release();
  return rc;
}

/* test hook: the device cut (lfr_cut.cuh) on one edge list, as graph.py::recursive_cut /
   lfr_cut.h recursive_cut_all with it as the only root: group_of[x] = the lowest node of x's group, x
   itself for a node no edge touches.  Edges (16 bytes: uint32 a, b, int64 w, lfr::CutEdge) must have
   a, b < n and a != b (a self-loop never leaves an oversized node's sub-problem in lfr_cut.h). */
typedef lfr::CutEdge lfr_cut_edge;
int lfr_debug_recursive_cut(const lfr_cut_edge* edges, uint64_t m, const uint32_t* node_weight, uint64_t n, uint32_t max_weight,
                            uint32_t* group_of) {
  lfr_options o;
  lfr_options_default(&o);
  LFR_TRY(select_device(o));
  if (m >= (1u << 30) || n >= (1u << 31)) return fail(LFR_EINVAL, "edge list too large");
  for (uint64_t i = 0; i < m; ++i)
    if (edges[i].a >= n || edges[i].b >= n || edges[i].a == edges[i].b) return fail(LFR_EINVAL, "cut edge out of range or a self-loop");
  for (uint64_t x = 0; x < n; ++x) group_of[x] = (uint32_t)x;
  if (m == 0) return LFR_OK;
  std::vector<uint32_t> a(m), b(m), sub(m, 0);
  std::vector<long long> w(m);
  for (uint64_t i = 0; i < m; ++i) {
    a[i] = edges[i].a;
    b[i] = edges[i].b;
    w[i] = edges[i].w;
  }
  CutLists E[2];
  DevBuf d_nw, d_label, tmp;
  uint32_t n_groups = 0;
  auto run = [&]() -> int {
    LFR_TRY(E[0].reserve(m));
    LFR_TRY(E[1].reserve(m));
    LFR_CUDA(cudaMemcpy(E[0].a.p, a.data(), 4 * m, cudaMemcpyHostToDevice));
    LFR_CUDA(cudaMemcpy(E[0].b.p, b.data(), 4 * m, cudaMemcpyHostToDevice));
    LFR_CUDA(cudaMemcpy(E[0].w.p, w.data(), 8 * m, cudaMemcpyHostToDevice));
    LFR_CUDA(cudaMemcpy(E[0].sub.p, sub.data(), 4 * m, cudaMemcpyHostToDevice));
    LFR_TRY(upload(&d_nw, node_weight, n, 0));
    LFR_TRY(upload(&d_label, group_of, n, 0));
    LFR_TRY(recursive_cut_on_device((uint32_t)n, E, (uint32_t)m, 1, d_nw.as<uint32_t>(), max_weight, 0, d_label.as<uint32_t>(), &n_groups,
                                    tmp, 0));
    LFR_CUDA(cudaMemcpy(group_of, d_label.p, 4 * n, cudaMemcpyDeviceToHost));
    return LFR_OK;
  };
  const int rc = run();
  d_nw.release(); d_label.release(); tmp.release();
  return rc;
}

}  // extern "C"
