// solver.cu — host side of libmcba.so: context, problem packing/upload, the trust-region driver and the
// extern "C" entry points declared in include/mcba.h.  No CPU fallback: everything numeric runs in the
// kernels of kernels.cuh / solver_kernels.cuh.
#include <cuda_runtime.h>
#include <cub/device/device_radix_sort.cuh>
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <cstdlib>
#include <string>
#include <chrono>
#include <functional>
#include <type_traits>
#include <memory>
#include <new>
#include <exception>
#include <vector>

#include "../../include/mcba.h"
#include "solver_kernels.cuh"
#include "linearize.cuh"
#include "lm_kernel.cuh"
#include "pack_kernels.cuh"
#include "table_kernels.cuh"
#include "pnp_kernels.cuh"
#include "intrinsics_kernels.cuh"
#include "pose_init_kernels.cuh"
#include "hand_eye_init_kernels.cuh"
#include "undistort_kernels.cuh"
#include "stereo_kernels.cuh"
#include "triangulate_kernels.cuh"

using namespace mcba;

namespace {

thread_local std::string g_create_error;

// A refusal or a CUDA error on the host: thrown by CK / CKL / REQUIRE, turned into a status and mcba_last_error's text only where an
// entry point returns (guarded)
struct Failure { int code; std::string msg; };

template <typename T>
struct DevBuf {
  T* p = nullptr;
  size_t n = 0;
  ~DevBuf() { release(); }
  void release() { if (p) cudaFree(p); p = nullptr; n = 0; }
  cudaError_t alloc(size_t count) {
    if (count <= n && p) return cudaSuccess;
    release();
    n = count ? count : 1;
    return cudaMalloc(&p, n * sizeof(T));
  }
};

// page-locked host staging (plain host memory on the test-suite's interpreter build, which has no pinned allocator)
cudaError_t host_alloc(uint8_t** p, size_t bytes) {
#ifdef MCBA_SIMT_BUILD
  *p = (uint8_t*)malloc(bytes);
  return *p ? cudaSuccess : cudaErrorMemoryAllocation;
#else
  return cudaMallocHost((void**)p, bytes);
#endif
}
void host_free(uint8_t* p) {
  if (!p) return;
#ifdef MCBA_SIMT_BUILD
  free(p);
#else
  cudaFreeHost(p);
#endif
}

// The parameter state is one block of doubles, [cam_rt 6C | board_rt 6B | frame_rt F fbs | intr kint C | he_rt 12 | board_pts 3BP] with
// fbs = max(fb, 6) doubles per frame: the current state (ctx->params) and the trial state (ctx->trial: what k_lm proposes, k_linearize
// evaluates) share it.  The board points come last: the uploads write them before the problem is set up, which zeroes everything in
// front of them.
struct StateLayout { size_t board, frame, intr, he, pts, len; };      // offsets of the blocks (cam_rt at 0) and the length

StateLayout state_layout(const mcba_problem_desc& d) {
  const size_t fbs = (d.optimize & MCBA_MOTION_ROLLING) ? 12 : 6;
  StateLayout L;
  L.board = 6 * (size_t)d.C; L.frame = L.board + 6 * (size_t)d.B; L.intr = L.frame + fbs * d.F;
  L.he = L.intr + (size_t)(5 + model_nd(d.model)) * d.C; L.pts = L.he + 12; L.len = L.pts + 3 * (size_t)d.B * d.P;
  return L;
}

// the parameter pointers of P into a state block
void set_state_pointers(DeviceProblem& P, double* base, const StateLayout& L) {
  P.cam_rt = base; P.board_rt = base + L.board; P.frame_rt = base + L.frame; P.intr = base + L.intr; P.he_rt = base + L.he; P.board_pts = base + L.pts;
}

// calls f(integral_constant<int, MODEL>, bool_constant<ROLL>) with the runtime camera model and rolling-shutter choice as constants
template <typename Fn>
void with_model(int model, bool roll, Fn&& f) {
  auto pick = [&](auto M) { if (roll) f(M, std::true_type{}); else f(M, std::false_type{}); };
  switch (model) {
    case MODEL_STANDARD: pick(std::integral_constant<int, MODEL_STANDARD>{}); break;
    case MODEL_RATIONAL: pick(std::integral_constant<int, MODEL_RATIONAL>{}); break;
    case MODEL_THIN_PRISM: pick(std::integral_constant<int, MODEL_THIN_PRISM>{}); break;
    case MODEL_TILTED: pick(std::integral_constant<int, MODEL_TILTED>{}); break;
    default: pick(std::integral_constant<int, MODEL_FISHEYE>{}); break;
  }
}

// calls f(integral_constant<int, LANES>) for the lanes of a triangulation group
template <typename Fn>
void with_lanes(int lanes, Fn&& f) {
  switch (lanes) {
    case 2: f(std::integral_constant<int, 2>{}); break;
    case 4: f(std::integral_constant<int, 4>{}); break;
    case 8: f(std::integral_constant<int, 8>{}); break;
    case 16: f(std::integral_constant<int, 16>{}); break;
    default: f(std::integral_constant<int, 32>{}); break;
  }
}

}  // namespace

struct mcba_ctx {
  int device = 0;
  cudaStream_t stream = nullptr;       // the stream every entry point works on
  cudaStream_t own_stream = nullptr;   // created by mcba_create; `stream` differs after mcba_set_stream
  std::string err;
  int rank = 0, world = 1;
  int launches = 0;
  int last_alpha_iters = 0;           // mcba_last_alpha_iterations
  int num_sms = 132;

  bool uploaded = false;
  DeviceProblem P{};
  // problem arrays
  DevBuf<double2> obs; DevBuf<uint16_t> pid; DevBuf<uint32_t> orig;
  DevBuf<int> view_start, view_cam, view_frame, view_board, frame_view_start;
  // the staged dense [C,F,B,P] table every upload packs from (the resident table's `valid` and observations): selection mask, pixels
  DevBuf<uint8_t> valid_mask, view_valid; DevBuf<double2> dense_pts; DevBuf<float2> dense_pts32; DevBuf<int> scan;
  cudaStream_t copy_stream = nullptr; cudaEvent_t copy_done = nullptr, copy_go = nullptr;      // observations in flight beside the view count
  DevBuf<PoseT> cam_T, frame_T, board_T;
  // parameter state (state_layout): current and trial
  StateLayout layout{};
  DevBuf<double> params, trial, pose_mats;
  // motion models: image heights (rolling), the hand-eye pose table and the fixed arm poses
  DevBuf<double> img_h; DevBuf<PoseT> he_T, arm_T;
  // solver buffers
  DevBuf<double> Hss, g, Hff, W, view_cost;
  // linearisation (linearize.cuh): per-(CTA, camera) records of the shared blocks, per-camera board partials, per-frame costs
  DevBuf<double> spart, bpart, frame_cost, sred;
  DevBuf<unsigned> cam_counter;
  // device-resident trust-region loop (lm_kernel.cuh)
  DevBuf<double> Spart, rpart, part_scale, part_quad, part_step;
  DevBuf<unsigned long long> lm_bar, peer_seq_dev, prof;
  bool profiling = false;      // MCBA_PROF=1 (with MCBA_GRAPH=0): phase timestamps of every k_lm launch on stderr
  DevBuf<mcba_log_row> dev_log;
  int lm_grid = 1, syrk_chunks = 1, syrk_cf = 8;
  bool use_graph = true;       // MCBA_GRAPH=0: the host launches one loop body at a time and reads the state after each
  struct SolveGraph { cudaGraphExec_t exec = nullptr; cudaGraph_t graph = nullptr; std::vector<char> key; cudaStream_t stream = nullptr; int body_launches = 0; } sg;
  bool graph_launched = false;
  int lin_grid = 1, lin_split = 1, lin_warps = LIN_WARPS;
  DevBuf<double> x, x_new, sinv, d, gh, gn, gq, piv, Y, Lf, zf, S, rhs, Linv;
  DevBuf<double> lin_cost, eval_cost;     // cost at the last linearisation (k_reduce_shared), cost of mcba_residuals
  DevBuf<SolverState> state;
  // NVLink peer-memory exchange of the solver kernel (lm_kernel.cuh LmPeer)
  double* peer_own = nullptr; int peer_cap = 0; bool peer_ready = false;
  double* peer_base[PEER_MAX_WORLD] = {nullptr};
  std::vector<void*> peer_opened;
  std::vector<int> perm;   // internal index -> canonical param_vec index
  // resident point table (mcba_table_*): inlier mask, sorted per-corner errors
  bool table = false; int table_selected = -1; bool errors_current = false;
  mcba_problem_desc table_desc{};
  int64_t n_valid = 0, n_inliers = 0;
  DevBuf<uint8_t> inlier_mask;
  DevBuf<double> err_valid, err_sorted, err_inl, err_inl_sorted, table_part, table_out;
  DevBuf<int64_t> table_ranks;
  DevBuf<unsigned char> sort_tmp;
  // batched pose initialisation (mcba_pnp_views): buffers kept between calls
  struct PnpBuffers {
    DevBuf<int64_t> start; DevBuf<int32_t> ids, grid, n; DevBuf<double2> xy, und; DevBuf<double> bp, in, pose, err; DevBuf<uint8_t> ok;
  } pnp;
  // intrinsic initialisation (mcba_intrinsic_init): used views, their homographies, K0
  struct IntrinsicBuffers {
    DevBuf<int32_t> used, cam_start, size; DevBuf<double> H, k0; DevBuf<uint8_t> hok;
  } intrinsic;
  // stereo initialisation (mcba_stereo_init): the intrinsics of the pair, relative poses, their sorted components, the start
  struct StereoBuffers {
    DevBuf<double> rel, sorted, rt0; DevBuf<uint8_t> both;
  } stereo;
  // pose-graph initialisation (mcba_pose_pairs / mcba_pose_times / mcba_pose_cluster): the table, the gathered rows, per-item results
  struct PoseInitBuffers {
    DevBuf<double> poses, cam, board, m1, m2, vecs, t; DevBuf<uint8_t> valid, mask, inl; DevBuf<PoseRow> rows;
    DevBuf<int64_t> start; DevBuf<int32_t> items, n_inl; DevBuf<char> work;
  } pinit;
  // non-overlapping camera initialisation (mcba_hand_eye_quads / mcba_hand_eye_vote)
  struct HandEyeInitBuffers {
    DevBuf<double> poses, X, Z, points, density; DevBuf<uint8_t> valid, ok; DevBuf<int32_t> quads, n_images, best; DevBuf<int64_t> start;
  } heinit;
  // applying a calibration (mcba_rectify_* / mcba_project_points): the cubic weight table, the resident maps of recent cameras
  // (fixed-point form, least recently used dropped first), the optional float map, points, and per-stream pinned staging for images
  struct UndistortMap {
    int model = -1, w = 0, h = 0; std::vector<double> cam; DevBuf<uint32_t> org; DevBuf<uint16_t> idx; uint64_t used = 0;
  };
  static constexpr int UND_STREAMS = 3, UND_MAX_MAPS = 64;
  struct UndistortBuffers {
    DevBuf<int32_t> tab; bool tab_ready = false;
    std::vector<std::unique_ptr<UndistortMap>> maps; uint64_t tick = 0;
    DevBuf<float2> fmap; DevBuf<double> pin, pout;
    cudaStream_t st[UND_STREAMS] = {}; cudaEvent_t done[UND_STREAMS] = {}, map_ready = nullptr;
    uint8_t* host_in[UND_STREAMS] = {}; uint8_t* host_out[UND_STREAMS] = {}; size_t host_in_cap = 0, host_out_cap = 0;
    DevBuf<uint8_t> dev_in[UND_STREAMS], dev_out[UND_STREAMS];
  } und;
  // triangulation (mcba_triangulate / mcba_triangulate_linear): the cameras, one chunk's inputs and outputs
  struct TriangulateBuffers {
    DevBuf<double> cams, poses, points, rms, lin; DevBuf<double2> px; DevBuf<uint8_t> valid, ok;
  } tri;
};

#define CK(call)                                                                                   \
  do {                                                                                             \
    cudaError_t e_ = (call);                                                                       \
    if (e_ != cudaSuccess) throw Failure{MCBA_ERR_CUDA, std::string(#call) + ": " + cudaGetErrorString(e_)}; \
  } while (0)
#define CKL()                                                                                      \
  do {                                                                                             \
    ctx->launches++;                                                                               \
    cudaError_t e_ = cudaGetLastError();                                                           \
    if (e_ != cudaSuccess) throw Failure{MCBA_ERR_CUDA, std::string("kernel launch: ") + cudaGetErrorString(e_)}; \
  } while (0)
// a macro, not a function: the message is built only when the check fails (it runs inside per-element loops)
#define REQUIRE(cond, code, msg)                                                                   \
  do { if (!(cond)) throw Failure{code, msg}; } while (0)

namespace {

// body() with whatever it throws as a status, its message in err: every C++ exception stops here, none crosses the C ABI
template <typename Fn>
int guarded(std::string& err, Fn&& body) {
  try { body(); return MCBA_OK; }
  catch (const Failure& f) { err = f.msg; return f.code; }
  catch (const std::bad_alloc&) { err = "host allocation failed (std::bad_alloc)"; }
  catch (const std::exception& e) { err = std::string("host exception: ") + e.what(); }
  catch (...) { err = "unknown host exception"; }
  return MCBA_ERR_CUDA;
}

// the boundary of an entry point: a null context, then the context's device, then the body
template <typename Fn>
int api(mcba_ctx* ctx, Fn&& body) {
  if (!ctx) return MCBA_ERR_ARG;
  return guarded(ctx->err, [&] { CK(cudaSetDevice(ctx->device)); body(); });
}

// full parameter state -> block-structured vector x (internal order)
__global__ void k_gather_params(DeviceProblem p, double* x, const double* cam_rt, const double* board_rt, const double* frame_rt, const double* intr) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= p.n) return;
  double v = 0.0;
  if (i >= p.n_s) v = frame_rt[i - p.n_s];
  else if (p.off_cp >= 0 && i >= p.off_cp && i < p.off_cp + 6 * p.C) v = cam_rt[i - p.off_cp];
  else if (p.off_bp >= 0 && i >= p.off_bp && i < p.off_bp + 6 * p.B) v = board_rt[i - p.off_bp];
  else if (p.off_in >= 0 && i >= p.off_in && i < p.off_in + p.kint * p.C) v = intr[i - p.off_in];
  else if (p.off_pt >= 0 && i >= p.off_pt && i < p.off_pt + 3 * p.B * p.P) v = p.board_pts[i - p.off_pt];
  else if (p.off_he >= 0 && i >= p.off_he && i < p.off_he + 12) v = p.he_rt[i - p.off_he];
  x[i] = v;
}
// x (internal order) -> trial state and its pose tables, one thread per item of make_trial_item (p: the current state)
__global__ void k_trial_state(DeviceProblem p, const double* x, double* trial, int n_items) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n_items) make_trial_item(p, x, trial, i);
}
// items of make_trial_item: poses, intrinsics per camera, padded board points, the hand-eye pair
int trial_items(const DeviceProblem& P) { return P.C + P.B + P.F * P.npf + P.C + P.B * P.P + 2; }

template <int MODE>
void launch_views(mcba_ctx* ctx, const DeviceProblem& P, const ViewKernelArgs& a) {
  const int blocks = std::max(1, std::min((P.V + VIEW_WARPS - 1) / VIEW_WARPS, ctx->num_sms * 8));
  const int th = VIEW_WARPS * 32;
  cudaStream_t s = ctx->stream;
  with_model(P.model, P.motion == MOTION_ROLLING, [&](auto M, auto R) {
    constexpr int MODEL = decltype(M)::value; constexpr bool ROLL = decltype(R)::value;
    k_views<MODEL, MODE, ROLL><<<blocks, th, 0, s>>>(P, a);
  });
  CKL();
}

// ---------------------------------------------------------------- linearisation (linearize.cuh)
size_t lin_smem_for(const DeviceProblem& P, int warps) {
  size_t bytes = 0;
  with_model(P.model, P.motion == MOTION_ROLLING, [&](auto M, auto R) {
    using S = LinShape<decltype(M)::value, decltype(R)::value>;
    bytes = sizeof(double) * lin_smem_doubles(S::NC, S::T, S::D, S::FB, S::NIN, P.B, S::NP, warps);
  });
  return bytes;
}
// one launch: H_ff, g_f, W_f, frame costs and the per-CTA records of the shared blocks at the (trial or current) state
void launch_linearize(mcba_ctx* ctx, const DeviceProblem& P, int loss, double f_scale) {
  if (P.F == 0) return;
  LinArgs a{}; a.loss = loss; a.f_scale = f_scale; a.split = ctx->lin_split;
  a.Hff = ctx->Hff.p; a.g = ctx->g.p; a.W = ctx->W.p; a.spart = ctx->spart.p; a.frame_cost = ctx->frame_cost.p;
  const size_t sm = lin_smem_for(P, ctx->lin_warps);
  const int th = ctx->lin_warps * 32;
  cudaStream_t s = ctx->stream;
  with_model(P.model, P.motion == MOTION_ROLLING, [&](auto M, auto R) {
    constexpr int MODEL = decltype(M)::value; constexpr bool ROLL = decltype(R)::value;
    k_linearize<MODEL, ROLL><<<ctx->lin_grid, th, sm, s>>>(P, a);
  });
  CKL();
}
// per-CTA records -> H_ss, g_s, cost (stores, fixed summation order)
void launch_reduce_shared(mcba_ctx* ctx, const DeviceProblem& P) {
  ReduceArgs r{}; r.spart = ctx->spart.p; r.nparts = P.F > 0 ? ctx->lin_grid : 0; r.Hss = ctx->Hss.p; r.g = ctx->g.p; r.bpart = ctx->bpart.p;
  r.frame_cost = ctx->frame_cost.p; r.F = P.F; r.cost_out = ctx->lin_cost.p; r.cam_counter = ctx->cam_counter.p; r.sred = ctx->sred.p;
  const size_t sm = sizeof(double) * reduce_smem_doubles(P.T, P.D);
  const int grid = P.C * reduce_slices(lin_record_doubles(P.T, P.D, P.B));
  if (P.motion == MOTION_ROLLING) k_reduce_shared<2><<<grid, RED_THREADS, sm, ctx->stream>>>(P, r);
  else k_reduce_shared<1><<<grid, RED_THREADS, sm, ctx->stream>>>(P, r);
  CKL();
}

// DeviceProblem view whose parameter pointers are the trial state
DeviceProblem with_state(const mcba_ctx* ctx, bool trial) {
  DeviceProblem P = ctx->P;
  if (trial) set_state_pointers(P, ctx->trial.p, ctx->layout);
  return P;
}

void prepare(mcba_ctx* ctx, const DeviceProblem& P) {
  const int np = P.C + P.B + P.F * P.npf + (P.motion == MOTION_HAND_EYE ? 2 : 0);
  k_prepare<<<(np + 127) / 128, 128, 0, ctx->stream>>>(P, P.cam_rt, P.board_rt, P.frame_rt);
  CKL();
}

// The normal equations and the cost at the (trial or current) state, whose pose tables must already describe it: k_linearize, its per-CTA
// records -> H_ss, g_s, cost (k_reduce_shared), then boards=True: the board-point blocks on top (k_point_blocks), then hand-eye: the
// hand-eye rows and columns from the frame blocks (k_fold_hand_eye, last: it reads the point rows of W_f)
void linearize(mcba_ctx* ctx, int loss, double f_scale, bool trial = false) {
  DeviceProblem P = with_state(ctx, trial);
  cudaStream_t s = ctx->stream;
  launch_linearize(ctx, P, loss, f_scale);
  if (P.off_pt >= 0) {         // k_point_blocks adds the point rows / columns (atomics): they start at zero
    CK(cudaMemsetAsync(ctx->Hss.p, 0, sizeof(double) * (size_t)P.n_s * P.n_s, s));
    CK(cudaMemsetAsync(ctx->g.p, 0, sizeof(double) * (size_t)std::max(P.n_s, 1), s));
  }
  launch_reduce_shared(ctx, P);
  if (P.off_pt >= 0 && P.V > 0) {
    ViewKernelArgs a{}; a.loss = loss; a.f_scale = f_scale;
    const int blocks = std::max(1, std::min((P.V + VIEW_WARPS - 1) / VIEW_WARPS, ctx->num_sms * 8));
    with_model(P.model, P.motion == MOTION_ROLLING, [&](auto M, auto R) {
      constexpr int MODEL = decltype(M)::value; constexpr int NP = decltype(R)::value ? 2 : 1;
      k_point_blocks<MODEL, NP><<<blocks, VIEW_WARPS * 32, 0, s>>>(P, a, ctx->Hss.p, ctx->W.p, ctx->g.p);
    });
    CKL();
  }
  if (P.off_he >= 0) {
    k_fold_hand_eye<<<P.n_s + 1, FOLD_THREADS, 0, s>>>(P, ctx->Hff.p, ctx->W.p, ctx->Hss.p, ctx->g.p);
    CKL();
  }
}

// cost at the (trial or current) state -> eval_cost
void trial_cost(mcba_ctx* ctx, int loss, double f_scale, bool trial) {
  DeviceProblem P = with_state(ctx, trial);
  ViewKernelArgs a{}; a.loss = loss; a.f_scale = f_scale; a.view_cost = ctx->view_cost.p;
  launch_views<MODE_COST>(ctx, P, a);
  k_sum_partials<<<1, 1024, 0, ctx->stream>>>(ctx->view_cost.p, P.V, 1, 1, ctx->eval_cost.p); CKL();
}

// ---------------------------------------------------------------- the device-resident trust-region loop (lm_kernel.cuh)
// trial parameter state := current state
void copy_state_to_trial(mcba_ctx* ctx) {
  CK(cudaMemcpyAsync(ctx->trial.p, ctx->params.p, sizeof(double) * ctx->layout.len, cudaMemcpyDeviceToDevice, ctx->stream));
}

// push vector x (internal order) into the trial state and rebuild the pose tables, as k_lm builds its trial states; trial == false:
// the trial state then becomes the current one.  The current state is only read, never updated in place: the derived hand-eye frame
// poses read he_rt while other items write its new value.
void set_state_from_x(mcba_ctx* ctx, const double* x, bool trial) {
  // make_trial_item writes every entry but he_rt of a problem without hand-eye and frame_rt of a hand-eye problem (derived frames):
  // those come from the copy
  copy_state_to_trial(ctx);
  const int items = trial_items(ctx->P);
  k_trial_state<<<(items + 127) / 128, 128, 0, ctx->stream>>>(ctx->P, x, ctx->trial.p, items);
  CKL();
  if (!trial) CK(cudaMemcpyAsync(ctx->params.p, ctx->trial.p, sizeof(double) * ctx->layout.len, cudaMemcpyDeviceToDevice, ctx->stream));
}

LmArgs make_lm_args(mcba_ctx* ctx, int log_cap) {
  const DeviceProblem& P = ctx->P;
  LmArgs a{};
  a.P = P;
  a.trial = ctx->trial.p; a.state_len = (int)ctx->layout.len;
  a.n = P.n; a.n_s = P.n_s; a.F = P.F; a.fb = P.fb;
  a.n_items = trial_items(P);
  a.Hss = ctx->Hss.p; a.Hff = ctx->Hff.p; a.W = ctx->W.p; a.g = ctx->g.p;
  a.frame_cost = ctx->frame_cost.p; a.lin_cost = ctx->lin_cost.p;
  a.x = ctx->x.p; a.x_new = ctx->x_new.p; a.sinv = ctx->sinv.p; a.d = ctx->d.p; a.gh = ctx->gh.p; a.gn = ctx->gn.p; a.gq = ctx->gq.p; a.piv = ctx->piv.p;
  a.Y = ctx->Y.p; a.Lf = ctx->Lf.p; a.zf = ctx->zf.p; a.S = ctx->S.p; a.rhs = ctx->rhs.p; a.Spart = ctx->Spart.p; a.rpart = ctx->rpart.p; a.Linv = ctx->Linv.p;
  a.syrk_chunks = ctx->syrk_chunks; a.syrk_cf = ctx->syrk_cf;
  a.part_scale = ctx->part_scale.p; a.part_quad = ctx->part_quad.p; a.part_step = ctx->part_step.p;
  a.st = ctx->state.p; a.log = ctx->dev_log.p; a.log_cap = log_cap; a.bar = ctx->lm_bar.p;
  a.peer.rank = ctx->rank; a.peer.world = ctx->world; a.peer.cap = ctx->peer_cap; a.peer.seq = ctx->peer_seq_dev.p;
  a.prof = ctx->profiling ? ctx->prof.p : nullptr;
  a.peer.timeout_cycles = (long long)40e9;          // ~20 s at 2 GHz: a rank that left the solve must not hang its peers' GPUs
  for (int r = 0; r < ctx->world && r < PEER_MAX_WORLD; r++) a.peer.base[r] = ctx->peer_base[r];
  return a;
}

void launch_lm(mcba_ctx* ctx, const LmArgs& a) {
  const size_t sm = sizeof(double) * lm_smem_doubles(ctx->P.n_s, ctx->P.fb);
  LmArgs args = a;
#ifdef MCBA_SIMT_BUILD
  if (ctx->P.tr_exact) {
    if (ctx->P.fb == 12) k_lm<12, true><<<ctx->lm_grid, LM_THREADS, sm, ctx->stream>>>(args); else k_lm<6, true><<<ctx->lm_grid, LM_THREADS, sm, ctx->stream>>>(args);
  } else {
    if (ctx->P.fb == 12) k_lm<12, false><<<ctx->lm_grid, LM_THREADS, sm, ctx->stream>>>(args); else k_lm<6, false><<<ctx->lm_grid, LM_THREADS, sm, ctx->stream>>>(args);
  }
  CKL();
#else
  // cooperative launch: every CTA of the grid is resident for the whole kernel (the grid barriers spin)
  void* params[] = {&args};
  const void* fn = ctx->P.tr_exact ? (ctx->P.fb == 12 ? (const void*)k_lm<12, true> : (const void*)k_lm<6, true>)
                                   : (ctx->P.fb == 12 ? (const void*)k_lm<12, false> : (const void*)k_lm<6, false>);
  CK(cudaLaunchCooperativeKernel(fn, dim3(ctx->lm_grid), dim3(LM_THREADS), params, sm, ctx->stream));
  ctx->launches++;
#endif
}

// one pass of the loop body: linearise the trial state, then accept / solve / step (k_lm)
void lm_body(mcba_ctx* ctx, int loss, double f_scale, const LmArgs& a) {
  linearize(ctx, loss, f_scale, true);
  launch_lm(ctx, a);
}

void run_lm_loop(mcba_ctx* ctx, int loss, double f_scale, int log_cap) {
  cudaStream_t s = ctx->stream;
  LmArgs a = make_lm_args(ctx, log_cap);
#ifndef MCBA_SIMT_BUILD
  if (ctx->use_graph) {
    // key of the cached graph: every launch parameter of the body (pointers, sizes, loss): the same problem solved again reuses it
    std::vector<char> key(sizeof(LmArgs) + sizeof(int) * 4 + sizeof(double));
    memcpy(key.data(), &a, sizeof(LmArgs));
    { char* q = key.data() + sizeof(LmArgs); memcpy(q, &loss, 4); memcpy(q + 4, &ctx->lin_grid, 4); memcpy(q + 8, &ctx->lm_grid, 4); { const int sw = ctx->lin_split * 16 + ctx->lin_warps; memcpy(q + 12, &sw, 4); } memcpy(q + 16, &f_scale, 8); }
    const int before = ctx->launches;
    if (!ctx->sg.exec || ctx->sg.key != key || ctx->sg.stream != s) {
      if (ctx->sg.exec) { cudaGraphExecDestroy(ctx->sg.exec); ctx->sg.exec = nullptr; }
      if (ctx->sg.graph) { cudaGraphDestroy(ctx->sg.graph); ctx->sg.graph = nullptr; }
      cudaGraph_t g; CK(cudaGraphCreate(&g, 0));
      ctx->sg.graph = g;
      cudaGraphConditionalHandle handle;
      CK(cudaGraphConditionalHandleCreate(&handle, g, 1, cudaGraphCondAssignDefault));
      cudaGraphNodeParams np = {cudaGraphNodeTypeConditional};
      np.conditional.handle = handle; np.conditional.type = cudaGraphCondTypeWhile; np.conditional.size = 1;
      cudaGraphNode_t node; CK(cudaGraphAddNode(&node, g, nullptr, 0, &np));
      cudaGraph_t body = np.conditional.phGraph_out[0];
      a.cond_handle = (unsigned long long)handle; a.use_cond = 1;
      // captured on the context's own stream (the caller's may be the legacy default stream, which cannot capture); the graph is
      // launched on the caller's stream
      cudaStream_t cap = ctx->own_stream;
      CK(cudaStreamSynchronize(s));
      CK(cudaStreamBeginCaptureToGraph(cap, body, nullptr, nullptr, 0, cudaStreamCaptureModeRelaxed));
      ctx->stream = cap;
      struct Capture {       // on every path, a throw from the body included: the context's stream back, the capture ended
        mcba_ctx* ctx; cudaStream_t s, cap; bool open = true;
        cudaError_t end() { open = false; ctx->stream = s; return cudaStreamEndCapture(cap, nullptr); }
        ~Capture() { if (open) end(); }
      } capture{ctx, s, cap};
      lm_body(ctx, loss, f_scale, a);
      const cudaError_t e = capture.end();
      REQUIRE(e == cudaSuccess, MCBA_ERR_CUDA, std::string("graph capture of the loop body: ") + cudaGetErrorString(e));
      CK(cudaGraphInstantiate(&ctx->sg.exec, g, 0));
      ctx->sg.key = key; ctx->sg.stream = s;
      ctx->sg.body_launches = ctx->launches - before;
    }
    ctx->launches = before;
    CK(cudaGraphLaunch(ctx->sg.exec, s));
    ctx->graph_launched = true;
    return;
  }
#endif
  // host-driven loop (the SIMT interpreter build; MCBA_GRAPH=0): same kernels, one state read per body
  ctx->graph_launched = false;
  SolverState h{};
  for (int it = 0; it < 2 * (log_cap + 8); it++) {      // (tr_solver='exact': a rejected trial costs a second pass, a relinearisation)
    lm_body(ctx, loss, f_scale, a);
    CK(cudaMemcpyAsync(&h, ctx->state.p, sizeof(h), cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    if (ctx->profiling) {
      unsigned long long t[16];
      CK(cudaMemcpy(t, ctx->prof.p, sizeof(t), cudaMemcpyDeviceToHost));
      fprintf(stderr, "[k_lm phases, us since phase A]");
      for (int q = 2; q <= 12; q++) fprintf(stderr, " %d:%.1f", q, t[q] >= t[1] && t[1] ? (t[q] - t[1]) * 1e-3 : -1.0);      // 11, 12: blocked Cholesky done, substitutions done
      fprintf(stderr, "\n");
      CK(cudaMemset(ctx->prof.p, 0, sizeof(t)));
    }
    if (h.done) break;
  }
}

// the current and trial parameter state of `desc` (kept when they already fit: a re-selected table keeps its state); returns where the
// uploads write the board points
double* alloc_state(mcba_ctx* ctx, const mcba_problem_desc* desc) {
  ctx->layout = state_layout(*desc);
  CK(ctx->params.alloc(ctx->layout.len)); CK(ctx->trial.alloc(ctx->layout.len));
  return ctx->params.p + ctx->layout.pts;
}

// dimensions, variable layout, permutation and every solver buffer that depends on (C,F,B,P,N,V)
void setup_problem(mcba_ctx* ctx, const mcba_problem_desc* desc, int64_t N, int V, bool keep_state = false) {
  const int C = desc->C, F = desc->F, B = desc->B, Pn = desc->P;
  DeviceProblem& P = ctx->P;
  P = DeviceProblem{};
  P.C = C; P.F = F; P.B = B; P.P = Pn; P.model = desc->model; P.nd = model_nd(desc->model);
  const int opt = desc->optimize;
  P.motion = (opt & MCBA_MOTION_ROLLING) ? MOTION_ROLLING : (opt & MCBA_MOTION_HAND_EYE) ? MOTION_HAND_EYE : MOTION_STATIC;
  P.npf = P.motion == MOTION_ROLLING ? 2 : 1;
  P.fb = P.motion == MOTION_ROLLING ? 12 : P.motion == MOTION_HAND_EYE ? 0 : 6;
  P.koff = 6 * P.npf;
  P.kint = 5 + P.nd; P.D = P.koff + 4 + P.nd; P.T = P.D * (P.D + 1) / 2 + P.D + 1;
  P.N = N; P.V = V;
  P.motion_on = ((opt & MCBA_OPT_MOTION) && P.fb > 0) ? 1 : 0;
  P.fix_aspect = (opt & MCBA_OPT_FIX_ASPECT) ? 1 : 0;
  int off = 0;
  P.off_cp = (opt & MCBA_OPT_CAMERA_POSES) ? off : -1; if (P.off_cp >= 0) off += 6 * C;
  P.off_bp = (opt & MCBA_OPT_BOARD_POSES) ? off : -1; if (P.off_bp >= 0) off += 6 * B;
  P.off_in = (opt & MCBA_OPT_CAMERAS) ? off : -1; if (P.off_in >= 0) off += P.kint * C;
  P.off_pt = (opt & MCBA_OPT_BOARDS) ? off : -1; if (P.off_pt >= 0) off += 3 * B * Pn;
  P.off_he = (P.motion == MOTION_HAND_EYE && (opt & MCBA_OPT_MOTION)) ? off : -1; if (P.off_he >= 0) off += 12;
  P.n_s = off; P.n_f = P.motion_on ? P.fb * F : 0; P.n = P.n_s + P.n_f;
  P.frame_blocks = (P.motion_on || P.off_he >= 0) ? 1 : 0;      // hand-eye: k_fold_hand_eye reads H_ff, W_f, g_f of the derived frames
  // internal -> canonical permutation: canonical = [cp | bp | motion | cameras]
  ctx->perm.assign((size_t)P.n, 0);
  {
    int canon = 0;
    if (P.off_cp >= 0) { for (int i = 0; i < 6 * C; i++) ctx->perm[(size_t)P.off_cp + i] = canon + i; canon += 6 * C; }
    if (P.off_bp >= 0) { for (int i = 0; i < 6 * B; i++) ctx->perm[(size_t)P.off_bp + i] = canon + i; canon += 6 * B; }
    // motion block of the reference vector: static [F][6]; rolling [start F x 6 | end F x 6] (rolling_frames.py:135-140) while the
    // solver keeps a frame's start | end adjacent; hand-eye [world_wrt_base 6 | gripper_wrt_camera 6] (hand_eye.py:76-81)
    if (P.motion_on) {
      for (int f = 0; f < F; f++) for (int j = 0; j < P.npf; j++) for (int k = 0; k < 6; k++)
        ctx->perm[(size_t)P.n_s + (size_t)f * P.fb + 6 * j + k] = canon + j * 6 * F + 6 * f + k;
      canon += P.fb * F;
    }
    if (P.off_he >= 0) { for (int i = 0; i < 12; i++) ctx->perm[(size_t)P.off_he + i] = canon + i; canon += 12; }
    if (P.off_in >= 0) { for (int i = 0; i < P.kint * C; i++) ctx->perm[(size_t)P.off_in + i] = canon + i; canon += P.kint * C; }
    if (P.off_pt >= 0) { for (int i = 0; i < 3 * B * Pn; i++) ctx->perm[(size_t)P.off_pt + i] = canon + i; canon += 3 * B * Pn; }
  }

  const size_t fbs = (size_t)std::max(P.fb, 6);      // doubles per frame in frame_rt and in the per-frame solver blocks
  alloc_state(ctx, desc);
  CK(ctx->cam_T.alloc(C)); CK(ctx->frame_T.alloc((size_t)std::max(F, 1) * P.npf)); CK(ctx->board_T.alloc(B));
  CK(ctx->img_h.alloc(C)); CK(ctx->he_T.alloc(2)); CK(ctx->arm_T.alloc(std::max(F, 1)));
  // solver buffers
  {
    // static frame -> CTA map (bit-reproducible partial sums): the smallest grid that keeps every CTA at ceil(F / resident CTAs) frames
    int split = 1;
    while (split < LIN_WARPS && C * split * 2 <= LIN_WARPS) split *= 2;      // few cameras: several warps share a view
    ctx->lin_split = split;
    // warps per CTA in {8, 4, 2}: the choice that keeps most warps resident per SM (shared memory: 227 KB minus ~4 KB per CTA;
    // registers: 128 per thread -> 16 warps) times how evenly the cameras spread over the CTA's warps (a warp owns cameras c == w mod warps;
    // the CTA meets at the end of every frame).  16 cameras x 5 boards (11 KB per warp): 2 CTAs of 8 warps; 4 of 4 score the same.
    int warps = LIN_WARPS;
    if (split == 1) {
      double best = -1.0;
      for (int wc = LIN_WARPS; wc >= 2; wc /= 2) {
        if (lin_smem_for(P, wc) > LIN_SMEM_MAX) continue;      // a CTA that large cannot be launched, even one per SM
        const size_t per_cta = lin_smem_for(P, wc) + 4 * 1024;
        const int occ = (int)std::min<size_t>((227 * 1024) / per_cta, (size_t)(16 / wc));
        if (occ < 1) continue;
        const double balance = (double)C / (double)(((C + wc - 1) / wc) * wc);
        const double score = occ * wc * balance;
        if (score > best + 1e-9) { best = score; warps = wc; }
      }
    }
    ctx->lin_warps = warps;
    {
      const size_t per_cta = lin_smem_for(P, warps) + 4 * 1024;
      const int occ = std::max(1, (int)std::min<size_t>((227 * 1024) / per_cta, (size_t)(16 / warps)));
      const int max_grid = ctx->num_sms * occ;
      const int per = (std::max(F, 1) + max_grid - 1) / max_grid;
      ctx->lin_grid = std::max(1, (std::max(F, 1) + per - 1) / per);
    }
    REQUIRE(lin_smem_for(P, warps) <= LIN_SMEM_MAX, MCBA_ERR_UNSUPPORTED, "too many boards for the linearisation kernel's shared memory");
    CK(ctx->spart.alloc((size_t)ctx->lin_grid * C * lin_record_doubles(P.T, P.D, B)));
    CK(ctx->bpart.alloc((size_t)C * B * 42));
    CK(ctx->sred.alloc((size_t)C * lin_record_doubles(P.T, P.D, B)));
    CK(ctx->cam_counter.alloc((size_t)C + 1)); CK(cudaMemsetAsync(ctx->cam_counter.p, 0, sizeof(unsigned) * ((size_t)C + 1), ctx->stream));
    CK(ctx->frame_cost.alloc((size_t)std::max(F, 1)));
  }
  CK(ctx->Hss.alloc((size_t)std::max(P.n_s, 1) * std::max(P.n_s, 1)));
  CK(cudaMemsetAsync(ctx->Hss.p, 0, sizeof(double) * (size_t)std::max(P.n_s, 1) * std::max(P.n_s, 1), ctx->stream));      // blocks no kernel writes (camera x other camera ...) stay zero
  const size_t ng = std::max<size_t>(std::max(P.n, 1), (size_t)P.n_s + (P.frame_blocks ? (size_t)F * fbs : 0));      // g_f of every frame block
  CK(ctx->g.alloc(ng));
  CK(cudaMemsetAsync(ctx->g.p, 0, sizeof(double) * ng, ctx->stream));
  CK(ctx->Hff.alloc((size_t)std::max(F, 1) * fbs * fbs));
  CK(ctx->W.alloc((size_t)std::max(F, 1) * std::max(P.n_s, 1) * fbs));
  {   // Y tile-major [row tile][frame][32][fb], rows beyond n_s stay zero (lm_kernel.cuh syrk_tile_acc)
    const size_t ny = (size_t)((std::max(P.n_s, 1) + SYRK_TILE - 1) / SYRK_TILE) * std::max(F, 1) * SYRK_TILE * fbs;
    CK(ctx->Y.alloc(ny)); CK(cudaMemsetAsync(ctx->Y.p, 0, sizeof(double) * ny, ctx->stream));
  }
  CK(ctx->Lf.alloc((size_t)std::max(F, 1) * fbs * fbs)); CK(ctx->zf.alloc((size_t)std::max(F, 1) * fbs));
  CK(ctx->view_cost.alloc((size_t)std::max(V, 1)));
  const size_t nn = (size_t)std::max(P.n, 1);
  CK(ctx->x.alloc(nn)); CK(ctx->x_new.alloc(nn)); CK(ctx->sinv.alloc(nn)); CK(ctx->d.alloc(nn)); CK(ctx->gh.alloc(nn)); CK(ctx->gn.alloc(nn)); CK(ctx->gq.alloc(nn));
  CK(ctx->S.alloc((size_t)std::max(P.n_s, 1) * std::max(P.n_s, 1))); CK(ctx->rhs.alloc((size_t)std::max(P.n_s, 1))); CK(ctx->piv.alloc((size_t)std::max(P.n_s, 1)));
  CK(ctx->Linv.alloc((size_t)((std::max(P.n_s, 1) + CHOL_NB - 1) / CHOL_NB) * CHOL_NB * CHOL_NB));
  CK(ctx->lin_cost.alloc(1)); CK(cudaMemsetAsync(ctx->lin_cost.p, 0, sizeof(double), ctx->stream));
  CK(ctx->eval_cost.alloc(1)); CK(cudaMemsetAsync(ctx->eval_cost.p, 0, sizeof(double), ctx->stream));
  // persistent trust-region kernel (lm_kernel.cuh): grid, frame chunks of the Schur SYRK, partial-sum records, barrier words
  {
    const int F_free = P.motion_on ? F : 0;
    // the whole machine except for toy problems: a phase's latency falls with the CTAs that share it, a grid barrier costs ~1 us either way
    ctx->lm_grid = (size_t)std::max(F_free, 1) * std::max(P.n_s, 1) >= 4096 ? ctx->num_sms : std::max(1, std::min(ctx->num_sms, 8));
    const int fbq = std::max(P.fb, 6), fr = syrk_fr(fbq);
    const int tiles = (std::max(P.n_s, 1) + SYRK_TILE - 1) / SYRK_TILE, npair = tiles * (tiles + 1) / 2;
    int chunks = std::max(1, std::min((F_free + fr - 1) / fr, ctx->lm_grid / std::max(1, npair)));
    const int cf = std::max(fr, ((std::max(F_free, 1) + chunks - 1) / chunks + fr - 1) / fr * fr);
    chunks = std::max(1, (F_free + cf - 1) / cf);
    ctx->syrk_chunks = chunks; ctx->syrk_cf = cf;
    REQUIRE(sizeof(double) * lm_smem_doubles(P.n_s, P.fb) <= 200 * 1024, MCBA_ERR_UNSUPPORTED, "reduced system too large for the trust-region kernel's shared memory");
    CK(ctx->Spart.alloc((size_t)chunks * std::max(P.n_s, 1) * std::max(P.n_s, 1)));
    CK(ctx->rpart.alloc((size_t)chunks * std::max(P.n_s, 1)));
    CK(ctx->part_scale.alloc((size_t)ctx->num_sms * 6));
    CK(ctx->part_step.alloc((size_t)ctx->num_sms * 2));
    CK(ctx->part_quad.alloc(8 + (size_t)(F + P.n_s + 2) * 5));
    CK(ctx->prof.alloc(16)); CK(cudaMemsetAsync(ctx->prof.p, 0, 16 * sizeof(unsigned long long), ctx->stream));
    CK(ctx->lm_bar.alloc(2)); CK(cudaMemsetAsync(ctx->lm_bar.p, 0, 2 * sizeof(unsigned long long), ctx->stream));
    if (!ctx->peer_seq_dev.p) { CK(ctx->peer_seq_dev.alloc(1)); CK(cudaMemsetAsync(ctx->peer_seq_dev.p, 0, sizeof(unsigned long long), ctx->stream)); }
  }
  CK(ctx->state.alloc(1));
  if (!keep_state) {     // a re-selection of the resident table (mcba_table_select) keeps the parameter state
    CK(cudaMemsetAsync(ctx->params.p, 0, sizeof(double) * ctx->layout.pts, ctx->stream));      // all but the uploaded board points
    // motion-model state: identity arm / hand-eye poses, unit image heights until mcba_set_rolling / mcba_set_hand_eye
    // (never read under static frames: no copies, no extra synchronisation on the BASELINE path)
    if (P.motion != MOTION_STATIC) {
      std::vector<double> ones((size_t)C, 1.0);
      CK(cudaMemcpyAsync(ctx->img_h.p, ones.data(), sizeof(double) * C, cudaMemcpyHostToDevice, ctx->stream));
      PoseT id{}; id.R[0] = id.R[4] = id.R[8] = 1.0;
      std::vector<PoseT> arms((size_t)std::max(F, 1), id);
      CK(cudaMemcpyAsync(ctx->arm_T.p, arms.data(), sizeof(PoseT) * arms.size(), cudaMemcpyHostToDevice, ctx->stream));
      CK(cudaStreamSynchronize(ctx->stream));
    }
  }

  P.obs = ctx->obs.p; P.pid = ctx->pid.p; P.orig = ctx->orig.p;
  P.view_start = ctx->view_start.p; P.view_cam = ctx->view_cam.p; P.view_frame = ctx->view_frame.p; P.view_board = ctx->view_board.p;
  P.frame_view_start = ctx->frame_view_start.p;
  set_state_pointers(P, ctx->params.p, ctx->layout);
  P.cam_T = ctx->cam_T.p; P.frame_T = ctx->frame_T.p; P.board_T = ctx->board_T.p;
  P.img_h = ctx->img_h.p; P.he_T = ctx->he_T.p; P.arm_T = ctx->arm_T.p;
}
// MCBA_PROF=1: host wall clock at checkpoints of the upload path, on stderr (no synchronisation is added: it times what the host waits for)
struct UploadClock {
  bool on; std::chrono::steady_clock::time_point t0;
  explicit UploadClock(bool enabled) : on(enabled), t0(std::chrono::steady_clock::now()) {}
  void mark(const char* what) { if (on) fprintf(stderr, "[upload] %-28s %8.3f ms\n", what, std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count()); }
};
void check_desc(const mcba_problem_desc* desc) {
  REQUIRE(desc->C > 0 && desc->F >= 0 && desc->B > 0 && desc->P > 0, MCBA_ERR_ARG, "bad problem dimensions");
  REQUIRE(desc->P <= 65535, MCBA_ERR_UNSUPPORTED, "more than 65535 points per board");
  REQUIRE(desc->model >= 0 && desc->model <= 4, MCBA_ERR_ARG, "unknown camera model");
  REQUIRE(!((desc->optimize & MCBA_MOTION_ROLLING) && (desc->optimize & MCBA_MOTION_HAND_EYE)), MCBA_ERR_ARG, "more than one motion model");
  REQUIRE((int64_t)desc->C * desc->F * desc->B * desc->P < ((int64_t)1 << 31), MCBA_ERR_UNSUPPORTED, "more than 2^31 table entries per rank");
}

// pack the resident dense table (ctx->dense_pts) under a device mask into the frame-major corner arrays the kernels read; returns the
// number of corners.  points_ready: event after which dense_pts holds the observations (they may still be in flight on the copy stream
// while the views are counted and scanned), or null
int64_t pack_dense(mcba_ctx* ctx, const mcba_problem_desc* desc, const uint8_t* d_mask, bool keep_state,
                   const uint8_t* d_view_valid = nullptr, cudaEvent_t points_ready = nullptr, bool points_f32 = false) {
  const int C = desc->C, F = desc->F, B = desc->B, Pn = desc->P;
  const int nv = C * F * B;
  cudaStream_t s = ctx->stream;
  CK(ctx->scan.alloc((size_t)3 * (nv + 1)));
  int* cnt_can = ctx->scan.p; int* cnt_fm = cnt_can + (nv + 1); int* flag_fm = cnt_fm + (nv + 1);
  int totals[2] = {0, 0};
  UploadClock clk(ctx->profiling);
  ctx->uploaded = false;      // the problem's buffers change from here on: set again only when setup_problem succeeds
  if (nv > 0) {
    k_pack_count<<<(unsigned)(((size_t)nv * 32 + 255) / 256), 256, 0, s>>>(d_mask, d_view_valid, C, F, B, Pn, cnt_can, cnt_fm, flag_fm); CKL();
    k_scan_exclusive<<<3, 1024, 0, s>>>(cnt_can, nv, nv + 1); CKL();      // cnt_can | cnt_fm | flag_fm
    CK(cudaMemcpyAsync(&totals[0], cnt_can + nv, sizeof(int), cudaMemcpyDeviceToHost, s));
    CK(cudaMemcpyAsync(&totals[1], flag_fm + nv, sizeof(int), cudaMemcpyDeviceToHost, s));
    clk.mark("pack: count/scan/d2h issued");
    CK(cudaStreamSynchronize(s));
    clk.mark("pack: totals on the host");
  }
  const int64_t N = totals[0]; const int V = totals[1];
  CK(ctx->obs.alloc((size_t)std::max<int64_t>(N, 1))); CK(ctx->pid.alloc((size_t)std::max<int64_t>(N, 1))); CK(ctx->orig.alloc((size_t)std::max<int64_t>(N, 1)));
  CK(ctx->view_start.alloc((size_t)V + 1)); CK(ctx->view_cam.alloc((size_t)std::max(V, 1))); CK(ctx->view_frame.alloc((size_t)std::max(V, 1))); CK(ctx->view_board.alloc((size_t)std::max(V, 1)));
  CK(ctx->frame_view_start.alloc((size_t)F + 1));
  if (points_ready) CK(cudaStreamWaitEvent(s, points_ready, 0));
  if (nv > 0) {
    PackOut o{ctx->obs.p, ctx->pid.p, ctx->orig.p, ctx->view_start.p, ctx->view_cam.p, ctx->view_frame.p, ctx->view_board.p,
              ctx->frame_view_start.p};
    const unsigned blocks = (unsigned)(((size_t)nv * 32 + 255) / 256);
    if (points_f32) { k_pack_scatter<float2><<<blocks, 256, 0, s>>>(d_mask, (const float2*)ctx->dense_pts32.p, C, F, B, Pn, cnt_can, cnt_fm, flag_fm, o); CKL(); }
    else { k_pack_scatter<double2><<<blocks, 256, 0, s>>>(d_mask, (const double2*)ctx->dense_pts.p, C, F, B, Pn, cnt_can, cnt_fm, flag_fm, o); CKL(); }
  } else {
    CK(cudaMemsetAsync(ctx->view_start.p, 0, sizeof(int), s)); CK(cudaMemsetAsync(ctx->frame_view_start.p, 0, sizeof(int) * (F + 1), s));
  }
  clk.mark("pack: scatter issued");
  setup_problem(ctx, desc, N, V, keep_state);
  clk.mark("pack: setup_problem done");
  CK(cudaStreamSynchronize(s));
  clk.mark("pack: final synchronise");
  ctx->uploaded = true;
  return N;
}

}  // namespace

// =====================================================================================================
extern "C" {

int mcba_version(void) { return 101; }

const char* mcba_last_error(const mcba_ctx* ctx) { return ctx ? ctx->err.c_str() : g_create_error.c_str(); }

int mcba_create(int device, mcba_ctx** out) {
  return guarded(g_create_error, [&] {
    REQUIRE(out, MCBA_ERR_ARG, "null output pointer");
    *out = nullptr;
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    REQUIRE(e == cudaSuccess && count > 0, MCBA_ERR_CUDA, std::string("no CUDA device: ") + cudaGetErrorString(e));
    REQUIRE(device >= 0 && device < count, MCBA_ERR_ARG, "device ordinal out of range");
    e = cudaSetDevice(device);
    REQUIRE(e == cudaSuccess, MCBA_ERR_CUDA, cudaGetErrorString(e));
    cudaDeviceProp prop;
    e = cudaGetDeviceProperties(&prop, device);
    REQUIRE(e == cudaSuccess, MCBA_ERR_CUDA, cudaGetErrorString(e));
    REQUIRE(prop.major == 9 && prop.minor == 0, MCBA_ERR_CUDA, "libmcba is built for sm_90a only (found sm_" + std::to_string(prop.major * 10 + prop.minor) + ")");
    std::unique_ptr<mcba_ctx> ctx(new mcba_ctx());
    ctx->device = device;
    ctx->num_sms = prop.multiProcessorCount;
    REQUIRE(cudaStreamCreateWithFlags(&ctx->own_stream, cudaStreamNonBlocking) == cudaSuccess, MCBA_ERR_CUDA, "cudaStreamCreate failed");
    ctx->stream = ctx->own_stream;
    { const char* e = getenv("MCBA_GRAPH"); if (e && std::string(e) == "0") ctx->use_graph = false; }
    { const char* e = getenv("MCBA_PROF"); if (e && std::string(e) == "1") { ctx->profiling = true; ctx->use_graph = false; } }
    for (int model = MODEL_STANDARD; model <= MODEL_TILTED; model++)
      for (bool roll : {false, true})
        with_model(model, roll, [](auto M, auto R) {
          cudaFuncSetAttribute(k_linearize<decltype(M)::value, decltype(R)::value>, cudaFuncAttributeMaxDynamicSharedMemorySize, LIN_SMEM_MAX);
        });
    cudaFuncSetAttribute(k_reduce_shared<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    cudaFuncSetAttribute(k_reduce_shared<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    cudaFuncSetAttribute(k_lm<6, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    cudaFuncSetAttribute(k_lm<12, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    cudaFuncSetAttribute(k_lm<6, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    cudaFuncSetAttribute(k_lm<12, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    cudaFuncSetAttribute(k_pose_align<PI_SMALL_THREADS, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, PI_SMALL_MAX * PI_ROW_BYTES);
    for (int model = MODEL_STANDARD; model <= MODEL_TILTED; model++)
      with_model(model, false, [](auto M, auto) {
        cudaFuncSetAttribute(k_triangulate<decltype(M)::value, 32>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                             (int)tri_smem((MCBA_TRI_MAX_CAMERAS + 31) / 32));
      });
    *out = ctx.release();
  });
}

void mcba_destroy(mcba_ctx* ctx) {
  if (!ctx) return;
  cudaSetDevice(ctx->device);
  cudaStreamSynchronize(ctx->stream);
#ifndef MCBA_SIMT_BUILD
  if (ctx->sg.exec) cudaGraphExecDestroy(ctx->sg.exec);
  if (ctx->sg.graph) cudaGraphDestroy(ctx->sg.graph);
#endif
  for (void* p : ctx->peer_opened) cudaIpcCloseMemHandle(p);
  if (ctx->peer_own) cudaFree(ctx->peer_own);
  if (ctx->copy_done) cudaEventDestroy(ctx->copy_done);
  if (ctx->copy_go) cudaEventDestroy(ctx->copy_go);
  if (ctx->copy_stream) cudaStreamDestroy(ctx->copy_stream);
  for (int i = 0; i < mcba_ctx::UND_STREAMS; i++) {
    auto& U = ctx->und;
    if (U.st[i]) { cudaStreamSynchronize(U.st[i]); cudaStreamDestroy(U.st[i]); }
    if (U.done[i]) cudaEventDestroy(U.done[i]);
    host_free(U.host_in[i]); host_free(U.host_out[i]);
  }
  if (ctx->und.map_ready) cudaEventDestroy(ctx->und.map_ready);
  cudaStream_t own = ctx->own_stream;
  delete ctx;                            // device buffers are freed by their destructors
  if (own) cudaStreamDestroy(own);
}

int mcba_set_stream(mcba_ctx* ctx, void* stream) {
  return api(ctx, [&] {
    CK(cudaStreamSynchronize(ctx->stream));          // nothing of ours may still be in flight on the stream we leave
    ctx->stream = (cudaStream_t)stream;              // NULL is the legacy default stream (what torch reports as stream 0)
  });
}

int mcba_comm_unique_id(mcba_ctx* ctx, char out_id[128]) {
  // kept for the shape of the API (rank 0 makes an id, the host broadcasts it): the exchanges of a solve run inside the solver kernel over
  // NVLink peer mappings (mcba_peer_export / mcba_peer_import), there is no library communicator to create
  return api(ctx, [&] {
    REQUIRE(out_id, MCBA_ERR_ARG, "null id buffer");
    memset(out_id, 0, 128);
    snprintf(out_id, 128, "mcba-peer-group");
  });
}

int mcba_comm_init(mcba_ctx* ctx, const char id_[128], int rank, int world) {
  return api(ctx, [&] {
    REQUIRE(id_, MCBA_ERR_ARG, "null id");
    REQUIRE(world >= 1 && world <= PEER_MAX_WORLD && rank >= 0 && rank < world, MCBA_ERR_ARG, "bad rank/world (1..16 ranks)");
    ctx->rank = rank; ctx->world = world; ctx->peer_ready = false;
  });
}

int mcba_peer_export(mcba_ctx* ctx, int64_t cap_doubles, char out_handle[64]) {
  return api(ctx, [&] {
    REQUIRE(out_handle, MCBA_ERR_ARG, "null handle buffer");
    REQUIRE(ctx->world > 1 && ctx->world <= PEER_MAX_WORLD, MCBA_ERR_STATE, "peer buffers need an initialised communicator with 2..16 ranks");
    REQUIRE(cap_doubles > 0 && cap_doubles < ((int64_t)1 << 30), MCBA_ERR_ARG, "bad peer slot capacity");
    REQUIRE(sizeof(cudaIpcMemHandle_t) == 64, MCBA_ERR_UNSUPPORTED, "unexpected cudaIpcMemHandle_t size");
    if (ctx->peer_own) { cudaFree(ctx->peer_own); ctx->peer_own = nullptr; }
    ctx->peer_ready = false; ctx->peer_cap = (int)cap_doubles;
    const size_t bytes = peer_buffer_doubles(ctx->world, ctx->peer_cap) * sizeof(double);
    CK(cudaMalloc(&ctx->peer_own, bytes));
    CK(cudaMemset(ctx->peer_own, 0, bytes));
    CK(cudaDeviceSynchronize());
    cudaIpcMemHandle_t h;
    CK(cudaIpcGetMemHandle(&h, ctx->peer_own));
    memcpy(out_handle, &h, 64);
  });
}

int mcba_peer_import(mcba_ctx* ctx, const char* handles /* world x 64 bytes, rank order */) {
  return api(ctx, [&] {
    REQUIRE(handles, MCBA_ERR_ARG, "null handles");
    REQUIRE(ctx->peer_own != nullptr, MCBA_ERR_STATE, "mcba_peer_export has not been called");
    for (int r = 0; r < ctx->world; r++) {
      if (r == ctx->rank) { ctx->peer_base[r] = ctx->peer_own; continue; }
      cudaIpcMemHandle_t h; memcpy(&h, handles + (size_t)r * 64, 64);
      void* p = nullptr;
      CK(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
      ctx->peer_base[r] = (double*)p; ctx->peer_opened.push_back(p);
    }
    // sequence number of the in-kernel exchanges (lm_kernel.cuh): starts at zero on every rank, advanced on the device
    CK(ctx->peer_seq_dev.alloc(1));
    CK(cudaMemset(ctx->peer_seq_dev.p, 0, sizeof(unsigned long long)));
    ctx->peer_ready = true;
  });
}

// ---------------------------------------------------------------------------------------------------------------
// Problem intake.  Every problem reaches the kernels the same way: a dense [C,F,B,P] table is staged on the device (ctx->valid_mask
// selects the corners, ctx->dense_pts or dense_pts32 holds their pixels) and pack_dense packs the selection frame-major
// (pack_kernels.cuh).  A caller's inputs are checked before any buffer of the context changes.

namespace {

bool all_finite(const double* p, size_t n) {
  for (size_t i = 0; i < n; i++) if (!std::isfinite(p[i])) return false;
  return true;
}

// The caller's detection lists: list w = (c*F+f)*B+b of the C*F*B views holds point ids det_ids[det_start[w]:det_start[w+1]] in [0, P) and
// their pixel corners det_xy (a CSR layout); the boards' id grids, when given, are at most 64 x 64.
void check_detections(const mcba_problem_desc* desc, const int64_t* det_start, const int32_t* det_ids, const double* det_xy,
                      const int32_t* board_grid) {
  const int nv = desc->C * desc->F * desc->B;
  const int64_t total = det_start[nv];
  REQUIRE(det_start[0] == 0 && total >= 0 && total < ((int64_t)1 << 31), MCBA_ERR_ARG, "bad detection offsets");
  REQUIRE(total == 0 || (det_ids && det_xy), MCBA_ERR_ARG, "null detection arrays");
  for (int w = 0; w < nv; w++) REQUIRE(det_start[w + 1] >= det_start[w], MCBA_ERR_ARG, "detection offsets are not a monotone CSR over C*F*B lists");
  for (int64_t i = 0; i < total; i++) REQUIRE(det_ids[i] >= 0 && det_ids[i] < desc->P, MCBA_ERR_ARG, "detection id outside [0, P)");
  for (int b = 0; board_grid && b < desc->B; b++)
    REQUIRE(board_grid[5 * b] > 0 && board_grid[5 * b + 1] > 0 && board_grid[5 * b + 2] > 0 && board_grid[5 * b] <= 64 && board_grid[5 * b + 1] <= 64,
            MCBA_ERR_UNSUPPORTED, "id grids are limited to 64 x 64 (bit masks of the occupied rows / columns)");
}

// detection lists in that layout -> ctx->pnp, with the id grids and the board points when given (the point table needs the lists only)
void stage_detections(mcba_ctx* ctx, const mcba_problem_desc* desc, const int64_t* det_start, const int32_t* det_ids, const double* det_xy,
                      const int32_t* board_grid, const double* board_points) {
  const int nv = desc->C * desc->F * desc->B, B = desc->B, Pn = desc->P;
  const int64_t total = det_start[nv];
  cudaStream_t s = ctx->stream;
  auto& pb = ctx->pnp;
  const size_t tot = (size_t)std::max<int64_t>(total, 1);
  CK(pb.start.alloc((size_t)nv + 1)); CK(pb.ids.alloc(tot)); CK(pb.xy.alloc(tot));
  CK(cudaMemcpyAsync(pb.start.p, det_start, sizeof(int64_t) * ((size_t)nv + 1), cudaMemcpyHostToDevice, s));
  if (total) {
    CK(cudaMemcpyAsync(pb.ids.p, det_ids, sizeof(int32_t) * (size_t)total, cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(pb.xy.p, det_xy, sizeof(double2) * (size_t)total, cudaMemcpyHostToDevice, s));
  }
  if (board_grid) {
    CK(pb.grid.alloc((size_t)B * 5));
    CK(cudaMemcpyAsync(pb.grid.p, board_grid, sizeof(int32_t) * (size_t)B * 5, cudaMemcpyHostToDevice, s));
  }
  if (board_points) {
    CK(pb.bp.alloc((size_t)B * Pn * 3));
    CK(cudaMemcpyAsync(pb.bp.p, board_points, sizeof(double) * (size_t)B * Pn * 3, cudaMemcpyHostToDevice, s));
  }
}

// k_pnp_views over the staged lists: one warp per list, poses under the intrinsics intr [C][kint] (device) of camera model `model`
void launch_pnp(mcba_ctx* ctx, const mcba_problem_desc* desc, int model, int kint, const double* intr) {
  auto& pb = ctx->pnp;
  PnpArgs a{};
  a.C = desc->C; a.F = desc->F; a.B = desc->B; a.P = desc->P; a.model = model; a.kint = kint; a.nv = desc->C * desc->F * desc->B;
  CK(pb.und.alloc(pb.ids.n)); CK(pb.pose.alloc((size_t)a.nv * 16)); CK(pb.err.alloc(a.nv)); CK(pb.n.alloc(a.nv)); CK(pb.ok.alloc(a.nv));
  a.det_start = pb.start.p; a.det_ids = pb.ids.p; a.det_xy = pb.xy.p; a.board_pts = pb.bp.p; a.intr = intr; a.grid = pb.grid.p;
  a.und = pb.und.p; a.poses = pb.pose.p; a.err = pb.err.p; a.npts = pb.n.p; a.valid = pb.ok.p; a.max_iters = 50;
  const int blocks = (a.nv + PNP_WARPS - 1) / PNP_WARPS;
  with_model(model, false, [&](auto M, auto) {
    constexpr int MODEL = decltype(M)::value;
    k_pnp_views<MODEL><<<blocks, PNP_WARPS * 32, 0, ctx->stream>>>(a);
  });
  CKL();
}

// Every upload starts here: whatever it refuses, and however late, it leaves no problem rather than a stale one (the entry points that
// need one fail with MCBA_ERR_STATE until an upload succeeds).
void drop_problem(mcba_ctx* ctx) {
  ctx->uploaded = false; ctx->table = false; ctx->table_selected = -1; ctx->errors_current = false;
}

// the dense table and the parameter state of `desc`; returns where the board points go
double* begin_intake(mcba_ctx* ctx, const mcba_problem_desc* desc, bool points_f32) {
  const size_t dense = std::max<size_t>((size_t)desc->C * desc->F * desc->B * desc->P, 1);
  CK(ctx->valid_mask.alloc(dense));
  if (points_f32) CK(ctx->dense_pts32.alloc(dense)); else CK(ctx->dense_pts.alloc(dense));
  return alloc_state(ctx, desc);
}

// A dense host table -> ctx->valid_mask (and ctx->view_valid), its points -> dense_pts or dense_pts32, the board points -> the state.
// Returns the event after which the points are on the device, or null.
cudaEvent_t stage_dense(mcba_ctx* ctx, const mcba_problem_desc* desc, const uint8_t* valid, const uint8_t* view_valid, const void* points,
                        int32_t point_type, const double* board_points) {
  REQUIRE(desc, MCBA_ERR_ARG, "null problem description");
  drop_problem(ctx);
  check_desc(desc);
  REQUIRE(valid && points && board_points, MCBA_ERR_ARG, "null dense table");
  REQUIRE(point_type == MCBA_POINTS_F64 || point_type == MCBA_POINTS_F32, MCBA_ERR_ARG, "unknown point type");
  const bool points_f32 = point_type == MCBA_POINTS_F32;
  const int nv = desc->C * desc->F * desc->B;
  const size_t dense = (size_t)nv * desc->P;
  double* bpts = begin_intake(ctx, desc, points_f32);
  if (view_valid) CK(ctx->view_valid.alloc((size_t)std::max(nv, 1)));
  cudaStream_t s = ctx->stream;
  UploadClock clk(ctx->profiling);
  cudaEvent_t points_ready = nullptr;
  // the mask (1 B/point) goes first on the solver's stream; the observations (16 B/point) follow on the copy stream while the views
  // are counted and scanned, and the scatter waits for them
  if (dense) CK(cudaMemcpyAsync(ctx->valid_mask.p, valid, dense, cudaMemcpyHostToDevice, s));
  if (dense && view_valid) CK(cudaMemcpyAsync(ctx->view_valid.p, view_valid, (size_t)nv, cudaMemcpyHostToDevice, s));
  // the small copies from pageable memory go BEFORE the table: such a copy returns when it is done, and behind 100 MB on the copy engine
  // it would hold the host back until the table has crossed the link -- with it the count / scan kernels that should run beside it
  CK(cudaMemcpyAsync(bpts, board_points, sizeof(double) * (size_t)desc->B * desc->P * 3, cudaMemcpyHostToDevice, s));
  if (dense) {
    if (!ctx->copy_stream) { CK(cudaStreamCreateWithFlags(&ctx->copy_stream, cudaStreamNonBlocking)); CK(cudaEventCreateWithFlags(&ctx->copy_done, cudaEventDisableTiming)); CK(cudaEventCreateWithFlags(&ctx->copy_go, cudaEventDisableTiming)); }
    CK(cudaEventRecord(ctx->copy_go, s));                          // work queued on `s` before this call may still read dense_pts
    CK(cudaStreamWaitEvent(ctx->copy_stream, ctx->copy_go, 0));
    if (points_f32) CK(cudaMemcpyAsync(ctx->dense_pts32.p, points, dense * sizeof(float2), cudaMemcpyHostToDevice, ctx->copy_stream));
    else CK(cudaMemcpyAsync(ctx->dense_pts.p, points, dense * sizeof(double2), cudaMemcpyHostToDevice, ctx->copy_stream));
    CK(cudaEventRecord(ctx->copy_done, ctx->copy_stream));
    points_ready = ctx->copy_done;
    clk.mark("upload: copies issued");
  }
  return points_ready;
}

// the staged table becomes the resident one: inliers = valid, pack `valid`, remember the description; returns the number of corners
int64_t table_finish(mcba_ctx* ctx, const mcba_problem_desc* desc, cudaEvent_t points_ready) {
  const size_t dense = (size_t)desc->C * desc->F * desc->B * desc->P;
  CK(ctx->inlier_mask.alloc(std::max<size_t>(dense, 1)));
  if (dense) CK(cudaMemcpyAsync(ctx->inlier_mask.p, ctx->valid_mask.p, dense, cudaMemcpyDeviceToDevice, ctx->stream));
  ctx->table_desc = *desc;
  const int64_t n = pack_dense(ctx, desc, ctx->valid_mask.p, false, nullptr, points_ready);
  ctx->table = true; ctx->table_selected = MCBA_TABLE_VALID;
  ctx->n_valid = n; ctx->n_inliers = n;
  return n;
}

size_t table_dense(const mcba_ctx* ctx) {
  const mcba_problem_desc& d = ctx->table_desc;
  return (size_t)d.C * d.F * d.B * d.P;
}

void sort_errors(mcba_ctx* ctx, const double* in, double* out, int64_t n) {
  size_t bytes = 0;
  CK(cub::DeviceRadixSort::SortKeys(nullptr, bytes, in, out, n, 0, 64, ctx->stream));
  CK(ctx->sort_tmp.alloc(bytes));
  bytes = ctx->sort_tmp.n;
  CK(cub::DeviceRadixSort::SortKeys(ctx->sort_tmp.p, bytes, in, out, n, 0, 64, ctx->stream));
  ctx->launches += 4;
}

}  // namespace

int mcba_upload_dense(mcba_ctx* ctx, const mcba_problem_desc* desc, const uint8_t* valid, const uint8_t* view_valid, const void* points,
                      int32_t point_type, const double* board_points, int64_t* n_corners) {
  return api(ctx, [&] {
    cudaEvent_t ready = stage_dense(ctx, desc, valid, view_valid, points, point_type, board_points);
    const int64_t n = pack_dense(ctx, desc, ctx->valid_mask.p, false, view_valid ? ctx->view_valid.p : nullptr, ready,
                                 point_type == MCBA_POINTS_F32);
    if (n_corners) *n_corners = n;
  });
}

// ---------------------------------------------------------------------------------------------------------------
// Resident point table (include/mcba.h "resident point table"): Calibration.adjust_outliers without host round trips.

int mcba_table_upload(mcba_ctx* ctx, const mcba_problem_desc* desc, const uint8_t* valid, const double* points,
                      const double* board_points, int64_t* n_valid) {
  return api(ctx, [&] {
    cudaEvent_t ready = stage_dense(ctx, desc, valid, nullptr, points, MCBA_POINTS_F64, board_points);
    const int64_t n = table_finish(ctx, desc, ready);
    if (n_valid) *n_valid = n;
  });
}

int mcba_table_from_detections(mcba_ctx* ctx, const mcba_problem_desc* desc, const int64_t* det_start, const int32_t* det_ids,
                               const double* det_xy, const double* board_points, int64_t* n_valid) {
  return api(ctx, [&] {
    REQUIRE(desc, MCBA_ERR_ARG, "null problem description");
    drop_problem(ctx);
    check_desc(desc);
    REQUIRE(det_start && board_points, MCBA_ERR_ARG, "null argument");
    check_detections(desc, det_start, det_ids, det_xy, nullptr);
    const int nv = desc->C * desc->F * desc->B;
    {   // a table entry holds one corner
      std::vector<int> list_of((size_t)desc->P, -1);
      for (int w = 0; w < nv; w++)
        for (int64_t i = det_start[w]; i < det_start[w + 1]; i++) {
          REQUIRE(list_of[det_ids[i]] != w, MCBA_ERR_ARG, "detection list " + std::to_string(w) + " repeats point id " + std::to_string(det_ids[i]));
          list_of[det_ids[i]] = w;
        }
    }
    const size_t dense = (size_t)nv * desc->P;
    cudaStream_t s = ctx->stream;
    double* bpts = begin_intake(ctx, desc, false);
    CK(cudaMemcpyAsync(bpts, board_points, sizeof(double) * (size_t)desc->B * desc->P * 3, cudaMemcpyHostToDevice, s));
    stage_detections(ctx, desc, det_start, det_ids, det_xy, nullptr, nullptr);
    if (dense) {
      CK(cudaMemsetAsync(ctx->valid_mask.p, 0, dense, s));
      CK(cudaMemsetAsync(ctx->dense_pts.p, 0, dense * sizeof(double2), s));    // fill_sparse leaves zeros where nothing was detected
    }
    if (det_start[nv] > 0) {      // the ids were checked above: k_table_fill's range guard never writes its flag
      auto& pb = ctx->pnp;
      k_table_fill<<<(unsigned)(((size_t)nv * 32 + 255) / 256), 256, 0, s>>>(pb.start.p, pb.ids.p, pb.xy.p, nv, desc->P, ctx->valid_mask.p, ctx->dense_pts.p, nullptr); CKL();
    }
    const int64_t n = table_finish(ctx, desc, nullptr);
    if (n_valid) *n_valid = n;
  });
}

// Batched board-pose initialisation (pnp_kernels.cuh): one warp per detection list.  Independent of the uploaded problem.
int mcba_pnp_views(mcba_ctx* ctx, const mcba_problem_desc* desc, const int64_t* det_start, const int32_t* det_ids, const double* det_xy,
                   const double* board_points, const double* intrinsics, const int32_t* board_grid,
                   double* poses, double* errors, int32_t* num_points, uint8_t* valid) {
  return api(ctx, [&] {
    REQUIRE(desc, MCBA_ERR_ARG, "null problem description");
    check_desc(desc);
    REQUIRE(det_start && board_points && intrinsics && board_grid && poses && errors && num_points && valid, MCBA_ERR_ARG, "null argument");
    const int nv = desc->C * desc->F * desc->B;
    if (nv == 0) return;
    check_detections(desc, det_start, det_ids, det_xy, board_grid);
    const int kint = 5 + model_nd(desc->model);
    cudaStream_t s = ctx->stream;
    auto& pb = ctx->pnp;
    stage_detections(ctx, desc, det_start, det_ids, det_xy, board_grid, board_points);
    CK(pb.in.alloc((size_t)desc->C * kint));
    CK(cudaMemcpyAsync(pb.in.p, intrinsics, sizeof(double) * (size_t)desc->C * kint, cudaMemcpyHostToDevice, s));
    launch_pnp(ctx, desc, desc->model, kint, pb.in.p);
    CK(cudaMemcpyAsync(poses, pb.pose.p, sizeof(double) * 16 * (size_t)nv, cudaMemcpyDeviceToHost, s));
    CK(cudaMemcpyAsync(errors, pb.err.p, sizeof(double) * (size_t)nv, cudaMemcpyDeviceToHost, s));
    CK(cudaMemcpyAsync(num_points, pb.n.p, sizeof(int32_t) * (size_t)nv, cudaMemcpyDeviceToHost, s));
    CK(cudaMemcpyAsync(valid, pb.ok.p, (size_t)nv, cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
  });
}

// Initialisation of single-camera intrinsic calibration (intrinsics_kernels.cuh): one homography per used view, K0 per camera
// (initIntrinsicParams2D), the initial per-view poses from k_pnp_views under K0 and zero distortion.  Independent of the uploaded problem.
int mcba_intrinsic_init(mcba_ctx* ctx, const mcba_problem_desc* desc, const int64_t* det_start, const int32_t* det_ids, const double* det_xy,
                        const double* board_points, const int32_t* board_grid, const int32_t* image_sizes, const uint8_t* view_use,
                        double* intrinsics, double* poses, uint8_t* ok) {
  return api(ctx, [&] {
    REQUIRE(desc, MCBA_ERR_ARG, "null problem description");
    check_desc(desc);
    REQUIRE(det_start && board_points && board_grid && image_sizes && view_use && intrinsics && poses && ok, MCBA_ERR_ARG, "null argument");
    const int C = desc->C, F = desc->F, B = desc->B, Pn = desc->P, nv = C * F * B;
    const bool fisheye = desc->model == MODEL_FISHEYE;
    const int kint = 5 + model_nd(desc->model);
    check_detections(desc, det_start, det_ids, det_xy, board_grid);
    for (int c = 0; c < C; c++) REQUIRE(image_sizes[2 * c] > 0 && image_sizes[2 * c + 1] > 0, MCBA_ERR_ARG, "image sizes must be positive");
    // OpenCV estimates an initial camera matrix only for planar targets (all object points at z = 0)
    for (size_t i = 0; i < (size_t)B * Pn; i++)
      REQUIRE(board_points[3 * i + 2] == 0.0, MCBA_ERR_UNSUPPORTED, "non-planar board (z != 0): the initial camera matrix needs planar targets");
    // used views grouped by camera, board-major inside a camera (the order of calibration_points, camera.py:229-235); the detection lists
    // of unused views are emptied, so that k_pnp_views sees only the used ones
    std::vector<int32_t> used, cam_start((size_t)C + 1, 0);
    for (int c = 0; c < C; c++) {
      for (int b = 0; b < B; b++) for (int f = 0; f < F; f++) { const int w = (c * F + f) * B + b; if (view_use[w]) used.push_back(w); }
      cam_start[(size_t)c + 1] = (int32_t)used.size();
    }
    std::vector<int64_t> start((size_t)nv + 1, 0);
    std::vector<int32_t> ids; std::vector<double> xy;
    for (int w = 0; w < nv; w++) {
      if (view_use[w]) {
        ids.insert(ids.end(), det_ids + det_start[w], det_ids + det_start[w + 1]);
        xy.insert(xy.end(), det_xy + 2 * det_start[w], det_xy + 2 * det_start[w + 1]);
      }
      start[(size_t)w + 1] = (int64_t)ids.size();
    }
    const int n_used = (int)used.size();
    cudaStream_t s = ctx->stream;
    auto& pb = ctx->pnp; auto& ib = ctx->intrinsic;
    stage_detections(ctx, desc, start.data(), ids.data(), xy.data(), board_grid, board_points);
    CK(ib.used.alloc((size_t)std::max(n_used, 1))); CK(ib.cam_start.alloc((size_t)C + 1)); CK(ib.size.alloc((size_t)C * 2));
    CK(ib.H.alloc((size_t)std::max(n_used, 1) * 9)); CK(ib.hok.alloc((size_t)std::max(n_used, 1))); CK(ib.k0.alloc((size_t)C * kint));
    if (n_used) CK(cudaMemcpyAsync(ib.used.p, used.data(), sizeof(int32_t) * used.size(), cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(ib.cam_start.p, cam_start.data(), sizeof(int32_t) * cam_start.size(), cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(ib.size.p, image_sizes, sizeof(int32_t) * (size_t)C * 2, cudaMemcpyHostToDevice, s));
    if (fisheye) {
      if (C) { k_fisheye_k0<<<(C + 127) / 128, 128, 0, s>>>(C, kint, ib.size.p, ib.k0.p); CKL(); }
    } else {
      if (n_used) {
        HomographyArgs h{};
        h.n_used = n_used; h.B = B; h.P = Pn; h.used = ib.used.p; h.det_start = pb.start.p; h.det_ids = pb.ids.p; h.det_xy = pb.xy.p;
        h.board_pts = pb.bp.p; h.H = ib.H.p; h.ok = ib.hok.p;
        k_view_homography<<<(n_used + HOMOG_WARPS - 1) / HOMOG_WARPS, HOMOG_WARPS * 32, 0, s>>>(h); CKL();
      }
      ZhangArgs z{};
      z.kint = kint; z.fix_aspect = (desc->optimize & MCBA_OPT_FIX_ASPECT) ? 1 : 0; z.cam_start = ib.cam_start.p; z.image_size = ib.size.p;
      z.H = ib.H.p; z.ok = ib.hok.p; z.intr = ib.k0.p;
      k_zhang_init<<<C, ZHANG_THREADS, 0, s>>>(z); CKL();
    }
    if (nv) {
      // zero distortion: the pinhole K0, or the fisheye K0 whose undistortion is exact at k = 0
      launch_pnp(ctx, desc, fisheye ? MODEL_FISHEYE : MODEL_STANDARD, kint, ib.k0.p);
      CK(cudaMemcpyAsync(poses, pb.pose.p, sizeof(double) * 16 * (size_t)nv, cudaMemcpyDeviceToHost, s));
      CK(cudaMemcpyAsync(ok, pb.ok.p, (size_t)nv, cudaMemcpyDeviceToHost, s));
    }
    CK(cudaMemcpyAsync(intrinsics, ib.k0.p, sizeof(double) * (size_t)C * kint, cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
  });
}

// Initialisation of stereo calibration (stereo_kernels.cuh): per-view poses of both cameras by k_pnp_views under the given intrinsics,
// then the median relative pose.  Independent of the uploaded problem.
int mcba_stereo_init(mcba_ctx* ctx, const mcba_problem_desc* desc, const int64_t* det_start, const int32_t* det_ids, const double* det_xy,
                     const double* board_points, const double* intrinsics, double* rt0, double* left_poses, uint8_t* ok) {
  return api(ctx, [&] {
    REQUIRE(desc, MCBA_ERR_ARG, "null problem description");
    check_desc(desc);
    REQUIRE(desc->C == 2 && desc->B == 1 && desc->F > 0, MCBA_ERR_ARG, "a stereo pair is 2 cameras, 1 board and at least one view");
    REQUIRE(det_start && board_points && intrinsics && rt0 && left_poses && ok, MCBA_ERR_ARG, "null argument");
    const int F = desc->F, Pn = desc->P;
    const int kint = 5 + model_nd(desc->model);
    const int32_t grid[5] = {1, 1, 1, 0, 0};           // the views are chosen already: no minimum-detections rule on the device
    check_detections(desc, det_start, det_ids, det_xy, grid);
    REQUIRE(all_finite(intrinsics, 2 * (size_t)kint), MCBA_ERR_NONFINITE, "non-finite camera parameter");
    // the per-view poses are the planar PnP of k_pnp_views
    for (size_t i = 0; i < (size_t)Pn; i++)
      REQUIRE(board_points[3 * i + 2] == 0.0, MCBA_ERR_UNSUPPORTED, "non-planar object points (z != 0): the initial view poses need planar targets");
    for (int c = 0; c < 2; c++)
      for (int f = 0; f < F; f++) {
        const int64_t n = det_start[c * F + f + 1] - det_start[c * F + f];
        REQUIRE(n >= 4, MCBA_ERR_DEGENERATE, "view " + std::to_string(f) + " has " + std::to_string(n) + " points: a view pose needs at least 4");
      }
    cudaStream_t s = ctx->stream;
    auto& pb = ctx->pnp; auto& sb = ctx->stereo;
    stage_detections(ctx, desc, det_start, det_ids, det_xy, grid, board_points);
    CK(pb.in.alloc((size_t)2 * kint));
    CK(cudaMemcpyAsync(pb.in.p, intrinsics, sizeof(double) * 2 * (size_t)kint, cudaMemcpyHostToDevice, s));
    launch_pnp(ctx, desc, desc->model, kint, pb.in.p);
    CK(sb.rel.alloc((size_t)6 * F)); CK(sb.sorted.alloc((size_t)6 * F)); CK(sb.rt0.alloc(6)); CK(sb.both.alloc((size_t)F));
    StereoStartArgs a{};
    a.F = F; a.poses = pb.pose.p; a.ok = pb.ok.p; a.rel = sb.rel.p; a.sorted = sb.sorted.p; a.rt0 = sb.rt0.p; a.both = sb.both.p;
    k_stereo_start<<<1, STEREO_THREADS, 0, s>>>(a); CKL();
    CK(cudaMemcpyAsync(rt0, sb.rt0.p, sizeof(double) * 6, cudaMemcpyDeviceToHost, s));
    CK(cudaMemcpyAsync(left_poses, pb.pose.p, sizeof(double) * 16 * (size_t)F, cudaMemcpyDeviceToHost, s));
    CK(cudaMemcpyAsync(ok, sb.both.p, (size_t)F, cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
  });
}

// Per-view sums of squared pixel errors and corner counts of the packed problem at the current parameters (intrinsics_kernels.cuh)
int mcba_view_errors(mcba_ctx* ctx, double* sumsq, int64_t* count) {
  return api(ctx, [&] {
    REQUIRE(sumsq && count, MCBA_ERR_ARG, "null argument");
    REQUIRE(ctx->uploaded, MCBA_ERR_STATE, "no problem uploaded");
    DeviceProblem P = with_state(ctx, false);
    const size_t nv = (size_t)P.C * P.F * P.B;
    if (nv == 0) return;
    prepare(ctx, P);
    DevBuf<double> ds; DevBuf<int64_t> dn;
    CK(ds.alloc(nv)); CK(dn.alloc(nv));
    cudaStream_t s = ctx->stream;
    CK(cudaMemsetAsync(ds.p, 0, sizeof(double) * nv, s)); CK(cudaMemsetAsync(dn.p, 0, sizeof(int64_t) * nv, s));
    if (P.V > 0) {
      ViewKernelArgs a{}; a.loss = MCBA_LOSS_LINEAR; a.f_scale = 1.0; a.view_cost = ctx->view_cost.p;
      launch_views<MODE_COST>(ctx, P, a);
      k_view_sumsq<<<(P.V + 255) / 256, 256, 0, s>>>(P, ctx->view_cost.p, ds.p, dn.p);
      CKL();
    }
    CK(cudaMemcpyAsync(sumsq, ds.p, sizeof(double) * nv, cudaMemcpyDeviceToHost, s));
    CK(cudaMemcpyAsync(count, dn.p, sizeof(int64_t) * nv, cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
  });
}

namespace {

void check_pose_dims(int32_t C, int32_t F, int32_t B) {
  REQUIRE(C > 0 && F > 0 && B > 0, MCBA_ERR_ARG, "bad pose table dimensions");
  REQUIRE((int64_t)C * F * B < ((int64_t)1 << 31), MCBA_ERR_UNSUPPORTED, "more than 2^31 views");
}

// Uploads the pose table, gathers the rows of every item (start: CSR row offsets, one segment per item) and runs align_transforms_robust
// on each (pose_init_kernels.cuh): items above PI_SMALL_MAX rows on the large-item kernel, the rest on the shared-memory one.  Leaves
// t [items][4][4], n_inl [items] and inl [rows] on the device.  vecs (host, [rows][6]) selects the cluster-only mode instead of rows.
void run_pose_align(mcba_ctx* ctx, int C, int F, int B, const double* poses, const uint8_t* valid, const double* cam, const double* board,
                    const std::vector<PoseRow>& rows, const std::vector<int64_t>& start, const double* vecs) {
  auto& pb = ctx->pinit;
  cudaStream_t s = ctx->stream;
  const int n_items = (int)start.size() - 1;
  const int64_t n_rows = start.back();
  PoseAlignArgs a{};
  a.C = C; a.F = F; a.B = B; a.n_rows = n_rows;
  const size_t nv = (size_t)C * F * B;
  if (poses) {
    CK(pb.poses.alloc(16 * nv)); CK(pb.valid.alloc(nv));
    CK(cudaMemcpyAsync(pb.poses.p, poses, sizeof(double) * 16 * nv, cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(pb.valid.p, valid, nv, cudaMemcpyHostToDevice, s));
    a.poses = pb.poses.p; a.valid = pb.valid.p;
  }
  if (cam) {
    CK(pb.cam.alloc(16 * (size_t)C)); CK(pb.board.alloc(16 * (size_t)B));
    CK(cudaMemcpyAsync(pb.cam.p, cam, sizeof(double) * 16 * C, cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(pb.board.p, board, sizeof(double) * 16 * B, cudaMemcpyHostToDevice, s));
    a.cam = pb.cam.p; a.board = pb.board.p;
  }
  const size_t nr = (size_t)std::max<int64_t>(n_rows, 1);
  CK(pb.start.alloc(start.size())); CK(pb.items.alloc((size_t)std::max(n_items, 1)));
  CK(pb.t.alloc(16 * (size_t)std::max(n_items, 1))); CK(pb.n_inl.alloc((size_t)std::max(n_items, 1))); CK(pb.inl.alloc(nr));
  CK(cudaMemcpyAsync(pb.start.p, start.data(), sizeof(int64_t) * start.size(), cudaMemcpyHostToDevice, s));
  a.row_start = pb.start.p; a.t = pb.t.p; a.n_inl = pb.n_inl.p; a.inl = pb.inl.p;
  if (vecs) {
    CK(pb.vecs.alloc(6 * nr));
    CK(cudaMemcpyAsync(pb.vecs.p, vecs, sizeof(double) * 6 * n_rows, cudaMemcpyHostToDevice, s));
    a.vecs = pb.vecs.p;
  } else if (n_rows) {
    CK(pb.rows.alloc(nr)); CK(pb.m1.alloc(12 * nr)); CK(pb.m2.alloc(12 * nr)); CK(pb.mask.alloc(nr));
    CK(cudaMemcpyAsync(pb.rows.p, rows.data(), sizeof(PoseRow) * n_rows, cudaMemcpyHostToDevice, s));
    a.rows = pb.rows.p; a.m1 = pb.m1.p; a.m2 = pb.m2.p; a.mask = pb.mask.p;
    const int grid = (int)std::min<int64_t>((n_rows + 255) / 256, 8 * (int64_t)ctx->num_sms);
    k_pose_gather<<<grid, 256, 0, s>>>(a); CKL();
  }
  // items by size class; the large ones first in the list
  std::vector<int32_t> order;
  int64_t large_rows = 0; int small_max = 0;
  for (int i = 0; i < n_items; i++) {
    const int64_t R = start[i + 1] - start[i];
    if (R > PI_SMALL_MAX) { order.push_back(i); large_rows += R; }
  }
  const int n_large = (int)order.size();
  for (int i = 0; i < n_items; i++) {
    const int64_t R = start[i + 1] - start[i];
    if (R > 0 && R <= PI_SMALL_MAX) { order.push_back(i); small_max = std::max(small_max, (int)R); }
  }
  if (order.empty()) return;
  CK(cudaMemcpyAsync(pb.items.p, order.data(), sizeof(int32_t) * order.size(), cudaMemcpyHostToDevice, s));
  if (n_large) {
    CK(pb.work.alloc((size_t)n_rows * PI_ROW_BYTES));
    a.work = pb.work.p; a.items = pb.items.p;
    k_pose_align<PI_LARGE_THREADS, true><<<n_large, PI_LARGE_THREADS, 0, s>>>(a); CKL();
  }
  const int n_small = (int)order.size() - n_large;
  if (n_small) {
    a.items = pb.items.p + n_large;
    k_pose_align<PI_SMALL_THREADS, false><<<n_small, PI_SMALL_THREADS, (size_t)small_max * PI_ROW_BYTES, s>>>(a); CKL();
  }
}

}  // namespace

// Relative poses of estimate_relative_poses (axis 0) / estimate_relative_poses_inv (axis 2), every (parent, child) pair in one launch chain
int mcba_pose_pairs(mcba_ctx* ctx, int32_t C, int32_t F, int32_t B, const double* poses, const uint8_t* valid, int32_t axis,
                    const int32_t* pairs, int32_t n_pairs, double* t, uint8_t* inliers, int32_t* n_inliers) {
  return api(ctx, [&] {
    check_pose_dims(C, F, B);
    REQUIRE(poses && valid, MCBA_ERR_ARG, "null pose table");
    REQUIRE(axis == 0 || axis == 2, MCBA_ERR_ARG, "axis must be 0 (cameras) or 2 (boards)");
    REQUIRE(n_pairs >= 0, MCBA_ERR_ARG, "negative pair count");
    REQUIRE(n_pairs == 0 || (pairs && t && inliers && n_inliers), MCBA_ERR_ARG, "null argument");
    const int n = axis == 0 ? C : B;
    const int64_t R = axis == 0 ? (int64_t)F * B : (int64_t)C * F;
    REQUIRE((int64_t)n_pairs * R < ((int64_t)1 << 31), MCBA_ERR_UNSUPPORTED, "more than 2^31 rows");
    for (int k = 0; k < n_pairs; k++)
      REQUIRE(pairs[2 * k] >= 0 && pairs[2 * k] < n && pairs[2 * k + 1] >= 0 && pairs[2 * k + 1] < n && pairs[2 * k] != pairs[2 * k + 1],
              MCBA_ERR_ARG, "pair index out of range");
    if (n_pairs == 0) return;
    REQUIRE(all_finite(poses, 16 * (size_t)C * F * B), MCBA_ERR_NONFINITE, "non-finite pose in the table");
    std::vector<PoseRow> rows((size_t)n_pairs * R);
    std::vector<int64_t> start((size_t)n_pairs + 1);
    for (int k = 0; k < n_pairs; k++) {
      const int p = pairs[2 * k], q = pairs[2 * k + 1];
      start[k] = k * R;
      PoseRow* o = rows.data() + k * R;
      if (axis == 0) {           // rows (f, b), f-major, of table[p] and table[q]
        for (int64_t r = 0; r < R; r++) o[r] = PoseRow{PI_ROW_PAIR, (int32_t)(p * R + r), (int32_t)(q * R + r), 0};
      } else {                   // rows (c, f), c-major, of the inverted table[:, :, p] and [:, :, q]
        for (int64_t r = 0; r < R; r++) o[r] = PoseRow{PI_ROW_PAIR_INV, (int32_t)(r * B + p), (int32_t)(r * B + q), 0};
      }
    }
    start[n_pairs] = (int64_t)n_pairs * R;
    run_pose_align(ctx, C, F, B, poses, valid, nullptr, nullptr, rows, start, nullptr);
    auto& pb = ctx->pinit;
    cudaStream_t s = ctx->stream;
    CK(cudaMemcpyAsync(t, pb.t.p, sizeof(double) * 16 * n_pairs, cudaMemcpyDeviceToHost, s));
    CK(cudaMemcpyAsync(n_inliers, pb.n_inl.p, sizeof(int32_t) * n_pairs, cudaMemcpyDeviceToHost, s));
    CK(cudaMemcpyAsync(inliers, pb.inl.p, (size_t)n_pairs * R, cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
  });
}

// Rig poses of initialise_poses (tables.py:370-375): per frame, align_transforms_robust over the (camera, board) rows, times = inv(t)
int mcba_pose_times(mcba_ctx* ctx, int32_t C, int32_t F, int32_t B, const double* poses, const uint8_t* valid, const double* cam_poses,
                    const uint8_t* cam_valid, const double* board_poses, const uint8_t* board_valid, double* times, uint8_t* times_valid) {
  return api(ctx, [&] {
    check_pose_dims(C, F, B);
    REQUIRE(poses && valid, MCBA_ERR_ARG, "null pose table");
    REQUIRE(cam_poses && cam_valid && board_poses && board_valid && times && times_valid, MCBA_ERR_ARG, "null argument");
    REQUIRE(all_finite(poses, 16 * (size_t)C * F * B) && all_finite(cam_poses, 16 * (size_t)C) && all_finite(board_poses, 16 * (size_t)B),
            MCBA_ERR_NONFINITE, "non-finite pose");
    std::vector<PoseRow> rows;
    std::vector<int64_t> start(1, 0);
    std::vector<int32_t> frame_of;
    for (int f = 0; f < F; f++) {
      const size_t r0 = rows.size();
      for (int c = 0; c < C; c++) for (int b = 0; b < B; b++) {
        const int v = (c * F + f) * B + b;
        if (cam_valid[c] && valid[v] && board_valid[b]) rows.push_back(PoseRow{PI_ROW_FRAME, v, 0, 0});
      }
      if (rows.size() > r0) { start.push_back((int64_t)rows.size()); frame_of.push_back(f); }
    }
    for (int f = 0; f < F; f++) {
      times_valid[f] = 0;
      for (int k = 0; k < 16; k++) times[16 * (size_t)f + k] = (k % 5 == 0) ? 1.0 : 0.0;
    }
    if (frame_of.empty()) return;
    run_pose_align(ctx, C, F, B, poses, valid, cam_poses, board_poses, rows, start, nullptr);
    std::vector<double> t(16 * frame_of.size());
    CK(cudaMemcpyAsync(t.data(), ctx->pinit.t.p, sizeof(double) * t.size(), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    for (size_t k = 0; k < frame_of.size(); k++) {
      double* o = times + 16 * (size_t)frame_of[k];
      pi_inv34(t.data() + 16 * k, o);
      o[12] = 0.0; o[13] = 0.0; o[14] = 0.0; o[15] = 1.0;
      times_valid[frame_of[k]] = 1;
    }
  });
}

// mean_robust's cluster alone (transform/common.py:6-13): per set of 6-vectors, the mask of the largest Ward cluster
int mcba_pose_cluster(mcba_ctx* ctx, int32_t n_sets, const int64_t* set_start, const double* vecs, uint8_t* mask) {
  return api(ctx, [&] {
    REQUIRE(n_sets >= 0 && (n_sets == 0 || set_start), MCBA_ERR_ARG, "null set offsets");
    if (n_sets == 0) return;
    REQUIRE(set_start[0] == 0, MCBA_ERR_ARG, "set offsets must start at 0");
    for (int k = 0; k < n_sets; k++) REQUIRE(set_start[k + 1] >= set_start[k], MCBA_ERR_ARG, "set offsets must not decrease");
    const int64_t N = set_start[n_sets];
    REQUIRE(N < ((int64_t)1 << 31), MCBA_ERR_UNSUPPORTED, "more than 2^31 vectors");
    REQUIRE(N == 0 || (vecs && mask), MCBA_ERR_ARG, "null argument");
    if (N == 0) return;
    REQUIRE(all_finite(vecs, 6 * (size_t)N), MCBA_ERR_NONFINITE, "non-finite vector");
    std::vector<int64_t> start(set_start, set_start + n_sets + 1);
    run_pose_align(ctx, 1, 1, 1, nullptr, nullptr, nullptr, nullptr, {}, start, vecs);
    CK(cudaMemcpyAsync(mask, ctx->pinit.inl.p, (size_t)N, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
  });
}

// One cv2.calibrateRobotWorldHandEye(SHAH) of HandEye.master_slave_pair (hand_eye/hand_eye.py:82-107) per quadruple, one CTA each
int mcba_hand_eye_quads(mcba_ctx* ctx, int32_t C, int32_t F, int32_t B, const double* poses, const uint8_t* valid, int32_t n_quads,
                        const int32_t* quads, double* X, double* Z, int32_t* n_images, uint8_t* ok) {
  return api(ctx, [&] {
    check_pose_dims(C, F, B);
    REQUIRE(poses && valid, MCBA_ERR_ARG, "null pose table");
    REQUIRE(n_quads >= 0, MCBA_ERR_ARG, "negative quadruple count");
    REQUIRE(n_quads == 0 || (quads && X && Z && n_images && ok), MCBA_ERR_ARG, "null argument");
    for (int k = 0; k < n_quads; k++) {
      const int32_t* q = quads + 4 * (size_t)k;
      REQUIRE(q[0] >= 0 && q[0] < C && q[1] >= 0 && q[1] < C && q[2] >= 0 && q[2] < B && q[3] >= 0 && q[3] < B, MCBA_ERR_ARG,
              "quadruple index out of range");
      REQUIRE(q[0] != q[1], MCBA_ERR_ARG, "quadruple with master == slave");
    }
    if (n_quads == 0) return;
    REQUIRE(all_finite(poses, 16 * (size_t)C * F * B), MCBA_ERR_NONFINITE, "non-finite pose in the table");
    auto& hb = ctx->heinit;
    cudaStream_t s = ctx->stream;
    const size_t nv = (size_t)C * F * B, nq = (size_t)n_quads;
    CK(hb.poses.alloc(16 * nv)); CK(hb.valid.alloc(nv));
    CK(hb.quads.alloc(4 * nq)); CK(hb.X.alloc(16 * nq)); CK(hb.Z.alloc(16 * nq)); CK(hb.n_images.alloc(nq)); CK(hb.ok.alloc(nq));
    CK(cudaMemcpyAsync(hb.poses.p, poses, sizeof(double) * 16 * nv, cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(hb.valid.p, valid, nv, cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(hb.quads.p, quads, sizeof(int32_t) * 4 * nq, cudaMemcpyHostToDevice, s));
    HandEyeArgs a{C, F, B, hb.poses.p, hb.valid.p, hb.quads.p, hb.X.p, hb.Z.p, hb.n_images.p, hb.ok.p};
    k_he_quads<<<n_quads, HE_THREADS, 0, s>>>(a); CKL();
    CK(cudaMemcpyAsync(X, hb.X.p, sizeof(double) * 16 * nq, cudaMemcpyDeviceToHost, s));
    CK(cudaMemcpyAsync(Z, hb.Z.p, sizeof(double) * 16 * nq, cudaMemcpyDeviceToHost, s));
    CK(cudaMemcpyAsync(n_images, hb.n_images.p, sizeof(int32_t) * nq, cudaMemcpyDeviceToHost, s));
    CK(cudaMemcpyAsync(ok, hb.ok.p, nq, cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
  });
}

// probabilistic_guess (hand_eye/helper.py:5-18) for every set: gaussian_kde densities at the points, and the argmax
int mcba_hand_eye_vote(mcba_ctx* ctx, int32_t n_sets, const int64_t* set_start, const double* points, double* density, int32_t* best) {
  return api(ctx, [&] {
    REQUIRE(n_sets >= 0 && (n_sets == 0 || (set_start && best)), MCBA_ERR_ARG, "null set offsets");
    if (n_sets == 0) return;
    REQUIRE(set_start[0] == 0, MCBA_ERR_ARG, "set offsets must start at 0");
    for (int k = 0; k < n_sets; k++) REQUIRE(set_start[k + 1] >= set_start[k], MCBA_ERR_ARG, "set offsets must not decrease");
    const int64_t N = set_start[n_sets];
    REQUIRE(N < ((int64_t)1 << 31), MCBA_ERR_UNSUPPORTED, "more than 2^31 points");
    REQUIRE(points && density, MCBA_ERR_ARG, "null argument");
    for (int k = 0; k < n_sets; k++)
      REQUIRE(set_start[k + 1] - set_start[k] > 3, MCBA_ERR_DEGENERATE,
              "set " + std::to_string(k) + " has " + std::to_string(set_start[k + 1] - set_start[k]) +
              " points: a 3-D kernel density estimate needs at least 4");
    REQUIRE(all_finite(points, 3 * (size_t)N), MCBA_ERR_NONFINITE, "non-finite point");
    auto& hb = ctx->heinit;
    cudaStream_t s = ctx->stream;
    CK(hb.start.alloc((size_t)n_sets + 1)); CK(hb.points.alloc(3 * (size_t)N)); CK(hb.density.alloc((size_t)N));
    CK(hb.best.alloc((size_t)n_sets));
    CK(cudaMemcpyAsync(hb.start.p, set_start, sizeof(int64_t) * (n_sets + 1), cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(hb.points.p, points, sizeof(double) * 3 * N, cudaMemcpyHostToDevice, s));
    HandEyeVoteArgs a{n_sets, hb.start.p, hb.points.p, hb.density.p, hb.best.p};
    k_he_vote<<<(n_sets + HE_VOTE_WARPS - 1) / HE_VOTE_WARPS, 32 * HE_VOTE_WARPS, 0, s>>>(a); CKL();
    CK(cudaMemcpyAsync(density, hb.density.p, sizeof(double) * N, cudaMemcpyDeviceToHost, s));
    CK(cudaMemcpyAsync(best, hb.best.p, sizeof(int32_t) * n_sets, cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    for (int k = 0; k < n_sets; k++)
      REQUIRE(best[k] >= 0, MCBA_ERR_DEGENERATE, "set " + std::to_string(k) + " has a singular covariance");
  });
}

namespace {

// the camera of the map and point entries: [fx fy cx cy skew dist...] with 5 + nd values of `model`
void check_camera(int32_t model, const double* camera) {
  REQUIRE(model >= MODEL_STANDARD && model <= MODEL_TILTED, MCBA_ERR_ARG, "unknown camera model");
  REQUIRE(camera, MCBA_ERR_ARG, "null camera");
  REQUIRE(all_finite(camera, 5 + (size_t)model_nd(model)), MCBA_ERR_NONFINITE, "non-finite camera parameter");
  REQUIRE(camera[0] != 0.0 && camera[1] != 0.0, MCBA_ERR_ARG, "zero focal length");
}

UndistortCamera make_camera(int model, const double* camera, int w, int h) {
  UndistortCamera c{};
  for (int i = 0; i < 5 + model_nd(model); i++) c.k[i] = camera[i];
  for (int i = 0; i < 9; i++) c.tilt[i] = (i % 4 == 0) ? 1.0 : 0.0;
  if (model == MODEL_TILTED) { double dMx[9], dMy[9]; tilt_matrices(camera[5 + 12], camera[5 + 13], c.tilt, dMx, dMy); }
  c.w = w; c.h = h;
  return c;
}

// the bicubic weight table, built on the context stream at first use
void ensure_cubic_table(mcba_ctx* ctx) {
  auto& U = ctx->und;
  if (U.tab_ready) return;
  CK(U.tab.alloc(16 * (size_t)UND_TAB_ENTRIES));
  k_cubic_table<<<(UND_TAB_ENTRIES + UND_THREADS - 1) / UND_THREADS, UND_THREADS, 0, ctx->stream>>>(U.tab.p); CKL();
  U.tab_ready = true;
}

// the resident fixed-point map of a key, computed on ctx->stream by launch(float map or null, org, idx) when it is not resident yet (or
// when the float map is asked for)
mcba_ctx::UndistortMap* resident_map(mcba_ctx* ctx, int model, const double* key, size_t nk, int w, int h, float* map_out,
                                     const std::function<void(float2*, uint32_t*, uint16_t*)>& launch) {
  auto& U = ctx->und;
  cudaStream_t s = ctx->stream;
  ensure_cubic_table(ctx);
  const size_t npx = (size_t)w * h;
  mcba_ctx::UndistortMap* m = nullptr;
  for (auto& e : U.maps)
    if (e->model == model && e->w == w && e->h == h && e->cam.size() == nk && std::memcmp(e->cam.data(), key, nk * sizeof(double)) == 0)
      m = e.get();
  if (!m || map_out) {
    if (!m) {
      if (U.maps.size() >= (size_t)mcba_ctx::UND_MAX_MAPS) {
        auto lru = std::min_element(U.maps.begin(), U.maps.end(), [](const auto& a, const auto& b) { return a->used < b->used; });
        CK(cudaStreamSynchronize(s));              // its buffers may still be read by work in flight
        U.maps.erase(lru);
      }
      U.maps.emplace_back(new mcba_ctx::UndistortMap());
      m = U.maps.back().get();
      CK(m->org.alloc(npx)); CK(m->idx.alloc(npx));
    }
    float2* f = nullptr;
    if (map_out) { CK(U.fmap.alloc(npx)); f = U.fmap.p; }
    launch(f, m->org.p, m->idx.p);
    m->model = -1;                                 // not usable until the launch is known to have gone in
    CKL();
    m->model = model; m->w = w; m->h = h; m->cam.assign(key, key + nk);
    if (map_out) {
      CK(cudaMemcpyAsync(map_out, f, sizeof(float2) * npx, cudaMemcpyDeviceToHost, s));
      CK(cudaStreamSynchronize(s));
    }
  }
  m->used = ++U.tick;
  return m;
}

// rr = P R and ir = rr^-1 (row-major 3x3) for the rectification entries; a singular or non-finite P R fails with MCBA_ERR_ARG
RectifyCamera make_rectify_camera(int model, const double* camera, const double* R, const double* P, int w, int h) {
  REQUIRE(R && P, MCBA_ERR_ARG, "null R or P");
  REQUIRE(all_finite(R, 9) && all_finite(P, 9), MCBA_ERR_NONFINITE, "non-finite R or P");
  RectifyCamera rc;
  rc.cam = make_camera(model, camera, w, h);
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) rc.rr[3 * i + j] = P[3 * i] * R[j] + P[3 * i + 1] * R[3 + j] + P[3 * i + 2] * R[6 + j];
  // Gauss-Jordan elimination with partial pivoting on [rr | I]
  double A[3][3], I[3][3];
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) { A[i][j] = rc.rr[3 * i + j]; I[i][j] = i == j ? 1.0 : 0.0; }
  for (int c = 0; c < 3; c++) {
    int p = c;
    for (int r = c + 1; r < 3; r++) if (std::fabs(A[r][c]) > std::fabs(A[p][c])) p = r;
    REQUIRE(A[p][c] != 0.0, MCBA_ERR_ARG, "P R is singular");
    for (int j = 0; j < 3; j++) { std::swap(A[c][j], A[p][j]); std::swap(I[c][j], I[p][j]); }
    for (int r = 0; r < 3; r++) {
      if (r == c) continue;
      const double f = A[r][c] / A[c][c];
      for (int j = 0; j < 3; j++) { A[r][j] -= f * A[c][j]; I[r][j] -= f * I[c][j]; }
    }
  }
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) rc.ir[3 * i + j] = I[i][j] / A[i][i];
  REQUIRE(all_finite(rc.ir, 9), MCBA_ERR_ARG, "P R is singular");
  return rc;
}

// the resident rectification map of a camera under (R, P) (k_rectify_map)
mcba_ctx::UndistortMap* rectification_map(mcba_ctx* ctx, int model, const double* camera, const double* R, const double* P, int w, int h,
                                          float* map_out) {
  const RectifyCamera rc = make_rectify_camera(model, camera, R, P, w, h);
  const size_t nk = 5 + (size_t)model_nd(model);
  std::vector<double> key(camera, camera + nk);
  key.insert(key.end(), R, R + 9); key.insert(key.end(), P, P + 9);
  cudaStream_t s = ctx->stream;
  return resident_map(ctx, model, key.data(), key.size(), w, h, map_out, [&](float2* f, uint32_t* org, uint16_t* idx) {
    with_model(model, false, [&](auto M, auto) { k_rectify_map<decltype(M)::value><<<h, UND_THREADS, 0, s>>>(rc, f, org, idx); });
  });
}

// cv2.remap(src[i], map, None, INTER_CUBIC) for n images through the resident map m of (width, height), host to host.  Chunks of images
// go through pinned staging on UND_STREAMS streams in turn: while the host copies one chunk into its staging buffer, earlier chunks are
// in flight (copy in, k_remap_cubic, copy out) on the other streams.
void remap_images(mcba_ctx* ctx, const mcba_ctx::UndistortMap* m, int32_t width, int32_t height, int32_t n, int32_t src_width,
                  int32_t src_height, int32_t channels, const uint8_t* const* src, uint8_t* const* dst) {
  auto& U = ctx->und;
  const size_t in_bytes = (size_t)src_width * src_height * channels, out_bytes = (size_t)width * height * channels;
  const size_t chunk_bytes = (size_t)8 << 20;
  const int per_chunk = (int)std::max<size_t>(1, std::min<size_t>((size_t)n, chunk_bytes / std::max(in_bytes, out_bytes)));
  const int n_chunks = (n + per_chunk - 1) / per_chunk;
  const int n_slots = std::min(mcba_ctx::UND_STREAMS, n_chunks);
  if (!U.map_ready) CK(cudaEventCreateWithFlags(&U.map_ready, cudaEventDisableTiming));
  if (U.host_in_cap < per_chunk * in_bytes || U.host_out_cap < per_chunk * out_bytes) {
    for (int i = 0; i < mcba_ctx::UND_STREAMS; i++) {
      if (U.st[i]) CK(cudaStreamSynchronize(U.st[i]));
      host_free(U.host_in[i]); host_free(U.host_out[i]);
      U.host_in[i] = U.host_out[i] = nullptr;
    }
    U.host_in_cap = std::max(U.host_in_cap, per_chunk * in_bytes);
    U.host_out_cap = std::max(U.host_out_cap, per_chunk * out_bytes);
  }
  for (int i = 0; i < n_slots; i++) {
    if (!U.st[i]) CK(cudaStreamCreateWithFlags(&U.st[i], cudaStreamNonBlocking));
    if (!U.done[i]) CK(cudaEventCreateWithFlags(&U.done[i], cudaEventDisableTiming));
    if (!U.host_in[i]) CK(host_alloc(&U.host_in[i], U.host_in_cap));
    if (!U.host_out[i]) CK(host_alloc(&U.host_out[i], U.host_out_cap));
    CK(U.dev_in[i].alloc(per_chunk * in_bytes)); CK(U.dev_out[i].alloc(per_chunk * out_bytes));
  }
  CK(cudaEventRecord(U.map_ready, ctx->stream));           // the map (and table) are written on the context stream
  for (int i = 0; i < n_slots; i++) CK(cudaStreamWaitEvent(U.st[i], U.map_ready, 0));
  RemapArgs a{};
  a.org = m->org.p; a.idx = m->idx.p; a.tab = U.tab.p; a.ws = src_width; a.hs = src_height; a.wm = width; a.hm = height;
  std::vector<int> pending(n_slots, -1);                    // chunk whose results a slot holds
  auto drain = [&](int slot) {
    const int ck = pending[slot];
    if (ck < 0) return;
    CK(cudaEventSynchronize(U.done[slot]));
    const int first = ck * per_chunk, cnt = std::min(per_chunk, n - first);
    for (int j = 0; j < cnt; j++) std::memcpy(dst[first + j], U.host_out[slot] + j * out_bytes, out_bytes);
    pending[slot] = -1;
  };
  for (int ck = 0; ck < n_chunks; ck++) {
    const int slot = ck % n_slots, first = ck * per_chunk, cnt = std::min(per_chunk, n - first);
    drain(slot);
    for (int j = 0; j < cnt; j++) std::memcpy(U.host_in[slot] + j * in_bytes, src[first + j], in_bytes);
    cudaStream_t s = U.st[slot];
    CK(cudaMemcpyAsync(U.dev_in[slot].p, U.host_in[slot], cnt * in_bytes, cudaMemcpyHostToDevice, s));
    a.src = U.dev_in[slot].p; a.dst = U.dev_out[slot].p;
    const dim3 grid((width + UND_THREADS - 1) / UND_THREADS, height, cnt);
    if (channels == 1) k_remap_cubic<1><<<grid, UND_THREADS, 0, s>>>(a);
    else k_remap_cubic<3><<<grid, UND_THREADS, 0, s>>>(a);
    CKL();
    CK(cudaMemcpyAsync(U.host_out[slot], U.dev_out[slot].p, cnt * out_bytes, cudaMemcpyDeviceToHost, s));
    CK(cudaEventRecord(U.done[slot], s));
    pending[slot] = ck;
  }
  for (int k = 0; k < n_slots; k++) drain((n_chunks + k) % n_slots);
}

// the checks every image entry makes before its map is looked up
void check_images(int32_t width, int32_t height, int32_t n, int32_t src_width, int32_t src_height, int32_t channels,
                  int32_t dtype, const uint8_t* const* src, uint8_t* const* dst) {
  REQUIRE(dtype == MCBA_IMAGE_UINT8, MCBA_ERR_ARG, "unsupported image dtype: only 8-bit unsigned images are remapped");
  REQUIRE(channels == 1 || channels == 3, MCBA_ERR_ARG, "unsupported channel count: 1 or 3 channels are remapped");
  REQUIRE(width > 0 && height > 0 && height <= 65535, MCBA_ERR_ARG, "map size out of range");
  REQUIRE(src_width > 0 && src_height > 0, MCBA_ERR_ARG, "empty source image");
  REQUIRE(n >= 0, MCBA_ERR_ARG, "negative image count");
  if (n == 0) return;
  REQUIRE(src && dst, MCBA_ERR_ARG, "null image list");
  for (int i = 0; i < n; i++) REQUIRE(src[i] && dst[i], MCBA_ERR_ARG, "null image " + std::to_string(i));
}

// point entries: copy in, one thread per point, copy out.  The projection of camera-frame points, or the rectification of pixels under
// R and P.
void run_points(mcba_ctx* ctx, bool project, int32_t model, const double* camera, int64_t n, const double* in, double* out,
                const double* R = nullptr, const double* P = nullptr) {
  check_camera(model, camera);
  RectifyCamera rc;
  if (!project) rc = make_rectify_camera(model, camera, R, P, 0, 0);
  REQUIRE(n >= 0, MCBA_ERR_ARG, "negative point count");
  if (n == 0) return;
  REQUIRE(in && out, MCBA_ERR_ARG, "null argument");
  auto& U = ctx->und;
  cudaStream_t s = ctx->stream;
  const size_t din = project ? 3 : 2;
  CK(U.pin.alloc(din * n)); CK(U.pout.alloc(2 * (size_t)n));
  CK(cudaMemcpyAsync(U.pin.p, in, sizeof(double) * din * n, cudaMemcpyHostToDevice, s));
  const UndistortCamera c = make_camera(model, camera, 0, 0);
  const unsigned blocks = (unsigned)((n + UND_THREADS - 1) / UND_THREADS);
  with_model(model, false, [&](auto M, auto) {
    constexpr int MODEL = decltype(M)::value;
    if (project) k_project_points<MODEL><<<blocks, UND_THREADS, 0, s>>>(c, n, U.pin.p, U.pout.p);
    else k_rectify_points<MODEL><<<blocks, UND_THREADS, 0, s>>>(rc, n, U.pin.p, U.pout.p);
  });
  CKL();
  CK(cudaMemcpyAsync(out, U.pout.p, sizeof(double) * 2 * n, cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
}

}  // namespace

// initUndistortRectifyMap(K, dist, R, P, (width, height)) of one camera, kept resident for mcba_rectify_images
int mcba_rectify_map(mcba_ctx* ctx, int32_t model, const double* camera, const double* R, const double* P, int32_t width, int32_t height,
                     float* map) {
  return api(ctx, [&] {
    check_camera(model, camera);
    REQUIRE(width > 0 && height > 0 && height <= 65535, MCBA_ERR_ARG, "map size out of range");
    rectification_map(ctx, model, camera, R, P, width, height, map);
    CK(cudaStreamSynchronize(ctx->stream));
  });
}

// cv2.remap(src[i], map, None, INTER_CUBIC) for n images of one camera through its rectification map, host to host (remap_images)
int mcba_rectify_images(mcba_ctx* ctx, int32_t model, const double* camera, const double* R, const double* P, int32_t width,
                        int32_t height, int32_t n, int32_t src_width, int32_t src_height, int32_t channels, int32_t dtype,
                        const uint8_t* const* src, uint8_t* const* dst) {
  return api(ctx, [&] {
    check_camera(model, camera);
    check_images(width, height, n, src_width, src_height, channels, dtype, src, dst);
    if (n == 0) return;
    const mcba_ctx::UndistortMap* m = rectification_map(ctx, model, camera, R, P, width, height, nullptr);
    remap_images(ctx, m, width, height, n, src_width, src_height, channels, src, dst);
  });
}

int mcba_rectify_points(mcba_ctx* ctx, int32_t model, const double* camera, const double* R, const double* P, int64_t n,
                        const double* pixels, double* rectified) {
  return api(ctx, [&] {
    REQUIRE(R && P, MCBA_ERR_ARG, "null R or P");
    run_points(ctx, false, model, camera, n, pixels, rectified, R, P);
  });
}

int mcba_project_points(mcba_ctx* ctx, int32_t model, const double* camera, int64_t n, const double* points, double* pixels) {
  return api(ctx, [&] { run_points(ctx, true, model, camera, n, points, pixels); });
}

// the fixed-point bicubic weights k_remap_cubic reads, int32[1024][16]
int mcba_remap_cubic_table(mcba_ctx* ctx, int32_t* table) {
  return api(ctx, [&] {
    REQUIRE(table, MCBA_ERR_ARG, "null table");
    auto& U = ctx->und;
    ensure_cubic_table(ctx);
    CK(cudaMemcpyAsync(table, U.tab.p, sizeof(int32_t) * 16 * UND_TAB_ENTRIES, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
  });
}

namespace {

// points of one chunk: the chunk's device memory, at `bytes` per point, within MCBA_TRI_CHUNK_BYTES
int64_t tri_chunk(int64_t N, size_t bytes) { return std::max<int64_t>(1, std::min<int64_t>(N, (int64_t)(MCBA_TRI_CHUNK_BYTES / bytes))); }

}  // namespace

// N-view triangulation (k_triangulate), chunk by chunk: per chunk the pixels and masks of every camera go in (one copy per camera), one
// launch, the points, flags and rms come out
int mcba_triangulate(mcba_ctx* ctx, int32_t model, int32_t C, const double* cameras, const double* poses, int64_t N,
                     const double* pixels, const uint8_t* valid, double* points, uint8_t* ok, double* rms) {
  return api(ctx, [&] {
    REQUIRE(model >= MODEL_STANDARD && model <= MODEL_TILTED, MCBA_ERR_ARG, "unknown camera model");
    REQUIRE(C >= 1 && C <= MCBA_TRI_MAX_CAMERAS, MCBA_ERR_ARG, "camera count out of range (1 .. " + std::to_string(MCBA_TRI_MAX_CAMERAS) + ")");
    REQUIRE(N >= 0, MCBA_ERR_ARG, "negative point count");
    REQUIRE(cameras && poses, MCBA_ERR_ARG, "null cameras or poses");
    const int kd = 5 + model_nd(model);
    for (int c = 0; c < C; c++) {
      try {
        check_camera(model, cameras + (size_t)kd * c);
      } catch (Failure& f) {
        f.msg = "camera " + std::to_string(c) + ": " + f.msg;
        throw;
      }
    }
    REQUIRE(all_finite(poses, 16 * (size_t)C), MCBA_ERR_NONFINITE, "non-finite camera pose");
    if (N == 0) return;
    REQUIRE(pixels && valid && points && ok && rms, MCBA_ERR_ARG, "null argument");
    auto& T = ctx->tri;
    cudaStream_t s = ctx->stream;
    std::vector<double> cams((size_t)TRI_KD * C, 0.0);
    for (int c = 0; c < C; c++) std::copy(cameras + (size_t)kd * c, cameras + (size_t)kd * (c + 1), cams.begin() + (size_t)TRI_KD * c);
    const int lanes = tri_lanes(C), nk = (C + lanes - 1) / lanes;
    const int64_t chunk = tri_chunk(N, (size_t)C * (sizeof(double2) + 1) + 4 * sizeof(double) + 1);
    CK(T.cams.alloc(cams.size())); CK(T.poses.alloc(16 * (size_t)C));
    CK(T.px.alloc((size_t)C * chunk)); CK(T.valid.alloc((size_t)C * chunk));
    CK(T.points.alloc(3 * (size_t)chunk)); CK(T.rms.alloc(chunk)); CK(T.ok.alloc(chunk));
    CK(cudaMemcpyAsync(T.cams.p, cams.data(), sizeof(double) * cams.size(), cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(T.poses.p, poses, sizeof(double) * 16 * C, cudaMemcpyHostToDevice, s));
    for (int64_t p0 = 0; p0 < N; p0 += chunk) {
      const int64_t n = std::min(chunk, N - p0);
      for (int c = 0; c < C; c++) {
        CK(cudaMemcpyAsync(T.px.p + (size_t)c * n, pixels + 2 * ((size_t)c * N + p0), sizeof(double2) * n, cudaMemcpyHostToDevice, s));
        CK(cudaMemcpyAsync(T.valid.p + (size_t)c * n, valid + (size_t)c * N + p0, n, cudaMemcpyHostToDevice, s));
      }
      TriArgs a{C, nk, n, T.cams.p, T.poses.p, T.px.p, T.valid.p, T.points.p, T.ok.p, T.rms.p};
      const unsigned blocks = (unsigned)((n * lanes + TRI_THREADS - 1) / TRI_THREADS);
      with_model(model, false, [&](auto M, auto) {
        with_lanes(lanes, [&](auto L) {
          k_triangulate<decltype(M)::value, decltype(L)::value><<<blocks, TRI_THREADS, tri_smem(nk), s>>>(a);
        });
      });
      CKL();
      CK(cudaMemcpyAsync(points + 3 * p0, T.points.p, sizeof(double) * 3 * n, cudaMemcpyDeviceToHost, s));
      CK(cudaMemcpyAsync(ok + p0, T.ok.p, n, cudaMemcpyDeviceToHost, s));
      CK(cudaMemcpyAsync(rms + p0, T.rms.p, sizeof(double) * n, cudaMemcpyDeviceToHost, s));
    }
    CK(cudaStreamSynchronize(s));
  });
}

// cv2.triangulatePoints (k_triangulate_linear), chunk by chunk
int mcba_triangulate_linear(mcba_ctx* ctx, const double* P1, const double* P2, int64_t N, const double* x1, const double* x2, double* out) {
  return api(ctx, [&] {
    REQUIRE(P1 && P2, MCBA_ERR_ARG, "null projection matrix");
    REQUIRE(all_finite(P1, 12) && all_finite(P2, 12), MCBA_ERR_NONFINITE, "non-finite projection matrix");
    REQUIRE(N >= 0, MCBA_ERR_ARG, "negative point count");
    if (N == 0) return;
    REQUIRE(x1 && x2 && out, MCBA_ERR_ARG, "null argument");
    auto& T = ctx->tri;
    cudaStream_t s = ctx->stream;
    const int64_t chunk = tri_chunk(N, 8 * sizeof(double));
    CK(T.lin.alloc(8 * (size_t)chunk));
    TriLinearArgs a{};
    for (int j = 0; j < 12; j++) { a.P[0][j] = P1[j]; a.P[1][j] = P2[j]; }
    for (int64_t p0 = 0; p0 < N; p0 += chunk) {
      const int64_t n = std::min(chunk, N - p0);
      double* dx = T.lin.p;                            // [x1 x; x1 y; x2 x; x2 y] of the chunk, then [4][n] out
      for (int r = 0; r < 2; r++) {
        CK(cudaMemcpyAsync(dx + r * n, x1 + r * N + p0, sizeof(double) * n, cudaMemcpyHostToDevice, s));
        CK(cudaMemcpyAsync(dx + (2 + r) * n, x2 + r * N + p0, sizeof(double) * n, cudaMemcpyHostToDevice, s));
      }
      a.n = n; a.x[0] = dx; a.x[1] = dx + 2 * n; a.out = dx + 4 * n;
      k_triangulate_linear<<<(unsigned)((2 * n + TRI_THREADS - 1) / TRI_THREADS), TRI_THREADS, tri_smem(1), s>>>(a);
      CKL();
      for (int j = 0; j < 4; j++) CK(cudaMemcpyAsync(out + j * N + p0, a.out + j * n, sizeof(double) * n, cudaMemcpyDeviceToHost, s));
    }
    CK(cudaStreamSynchronize(s));
  });
}

int mcba_table_download(mcba_ctx* ctx, uint8_t* valid, double* points) {
  return api(ctx, [&] {
    REQUIRE(ctx->table, MCBA_ERR_STATE, "no resident table (mcba_table_upload / mcba_table_from_detections)");
    const size_t dense = table_dense(ctx);
    if (valid && dense) CK(cudaMemcpyAsync(valid, ctx->valid_mask.p, dense, cudaMemcpyDeviceToHost, ctx->stream));
    if (points && dense) CK(cudaMemcpyAsync(points, ctx->dense_pts.p, dense * sizeof(double2), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
  });
}

int mcba_table_set_inliers(mcba_ctx* ctx, const uint8_t* mask) {
  return api(ctx, [&] {
    REQUIRE(ctx->table, MCBA_ERR_STATE, "no resident table (mcba_table_upload / mcba_table_from_detections)");
    const size_t dense = table_dense(ctx);
    if (dense) {
      if (mask) {
        CK(cudaMemcpyAsync(ctx->inlier_mask.p, mask, dense, cudaMemcpyHostToDevice, ctx->stream));
        k_mask_and<<<(unsigned)((dense + 255) / 256), 256, 0, ctx->stream>>>(ctx->inlier_mask.p, ctx->valid_mask.p, dense, ctx->inlier_mask.p); CKL();
      } else {
        CK(cudaMemcpyAsync(ctx->inlier_mask.p, ctx->valid_mask.p, dense, cudaMemcpyDeviceToDevice, ctx->stream));
      }
    }
    CK(cudaStreamSynchronize(ctx->stream));      // the host mask is borrowed only for the call
    ctx->errors_current = false;
    if (ctx->table_selected == MCBA_TABLE_INLIERS) ctx->table_selected = -1;     // the packed set no longer matches the mask
  });
}

int mcba_table_get_inliers(mcba_ctx* ctx, uint8_t* mask) {
  return api(ctx, [&] {
    REQUIRE(mask, MCBA_ERR_ARG, "null mask");
    REQUIRE(ctx->table, MCBA_ERR_STATE, "no resident table (mcba_table_upload / mcba_table_from_detections)");
    const size_t dense = table_dense(ctx);
    if (dense) CK(cudaMemcpyAsync(mask, ctx->inlier_mask.p, dense, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
  });
}

namespace {

// the resident table's corners under `which` become the packed problem (kept when already selected); returns their number
int64_t select_table(mcba_ctx* ctx, int which) {
  REQUIRE(ctx->table, MCBA_ERR_STATE, "no resident table (mcba_table_upload / mcba_table_from_detections)");
  REQUIRE(which == MCBA_TABLE_VALID || which == MCBA_TABLE_INLIERS, MCBA_ERR_ARG, "unknown table selection");
  if (ctx->table_selected == which) return ctx->P.N;
  ctx->errors_current = false;
  const uint8_t* m = which == MCBA_TABLE_VALID ? ctx->valid_mask.p : ctx->inlier_mask.p;
  ctx->table_selected = -1;      // until the packing succeeds
  const int64_t n = pack_dense(ctx, &ctx->table_desc, m, true);
  ctx->table_selected = which;
  if (which == MCBA_TABLE_INLIERS) ctx->n_inliers = n;
  return n;
}

}  // namespace

int mcba_table_select(mcba_ctx* ctx, int which, int64_t* n_corners) {
  return api(ctx, [&] {
    const int64_t n = select_table(ctx, which);
    if (n_corners) *n_corners = n;
  });
}

int mcba_table_errors(mcba_ctx* ctx, mcba_table_stats* stats) {
  return api(ctx, [&] {
    select_table(ctx, MCBA_TABLE_VALID);
    const DeviceProblem P = with_state(ctx, false);
    cudaStream_t s = ctx->stream;
    const int64_t N = P.N;
    double sums[3] = {0.0, 0.0, 0.0};
    if (N > 0) {
      CK(ctx->err_valid.alloc((size_t)N)); CK(ctx->err_sorted.alloc((size_t)N));
      CK(ctx->err_inl.alloc((size_t)N)); CK(ctx->err_inl_sorted.alloc((size_t)N));
      CK(ctx->table_part.alloc((size_t)3 * P.V + 3));
      prepare(ctx, P);
      ViewKernelArgs a{}; a.err = ctx->err_valid.p;
      launch_views<MODE_ERROR>(ctx, P, a);
      const int blocks = std::max(1, std::min((P.V + TABLE_WARPS - 1) / TABLE_WARPS, ctx->num_sms * 8));
      k_table_stats<<<blocks, TABLE_WARPS * 32, 0, s>>>(P, ctx->err_valid.p, ctx->inlier_mask.p, ctx->err_inl.p, ctx->table_part.p); CKL();
      double* d_sums = ctx->table_part.p + (size_t)3 * P.V;
      k_sum_partials<<<1, 1024, 0, s>>>(ctx->table_part.p, P.V, 3, 3, d_sums); CKL();
      CK(cudaMemcpyAsync(sums, d_sums, sizeof(sums), cudaMemcpyDeviceToHost, s));
      sort_errors(ctx, ctx->err_valid.p, ctx->err_sorted.p, N);
      sort_errors(ctx, ctx->err_inl.p, ctx->err_inl_sorted.p, N);
      CK(cudaStreamSynchronize(s));
    }
    ctx->n_valid = N; ctx->n_inliers = (int64_t)llround(sums[2]);
    ctx->errors_current = true;
    if (stats) { stats->n_valid = N; stats->n_inliers = ctx->n_inliers; stats->sumsq_valid = sums[0]; stats->sumsq_inliers = sums[1]; }
  });
}

int mcba_table_error_ranks(mcba_ctx* ctx, int which, const int64_t* ranks, int32_t n, double* out) {
  return api(ctx, [&] {
    REQUIRE(n <= 0 || (ranks && out), MCBA_ERR_ARG, "null ranks or output");
    REQUIRE(ctx->table && ctx->errors_current, MCBA_ERR_STATE, "mcba_table_errors has not run since the parameters or the selection changed");
    REQUIRE(which == MCBA_TABLE_VALID || which == MCBA_TABLE_INLIERS, MCBA_ERR_ARG, "unknown table selection");
    if (n <= 0) return;
    const int64_t count = which == MCBA_TABLE_VALID ? ctx->n_valid : ctx->n_inliers;
    for (int i = 0; i < n; i++) REQUIRE(ranks[i] >= 0 && ranks[i] < count, MCBA_ERR_ARG, "error rank out of range");
    CK(ctx->table_ranks.alloc((size_t)n)); CK(ctx->table_out.alloc((size_t)n));
    CK(cudaMemcpyAsync(ctx->table_ranks.p, ranks, sizeof(int64_t) * n, cudaMemcpyHostToDevice, ctx->stream));
    k_gather_ranks<<<(n + 127) / 128, 128, 0, ctx->stream>>>(which == MCBA_TABLE_VALID ? ctx->err_sorted.p : ctx->err_inl_sorted.p,
                                                           ctx->table_ranks.p, n, ctx->table_out.p); CKL();
    CK(cudaMemcpyAsync(out, ctx->table_out.p, sizeof(double) * n, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
  });
}

int mcba_table_count_below(mcba_ctx* ctx, int which, const double* thresholds, int32_t n, int64_t* counts) {
  return api(ctx, [&] {
    REQUIRE(n <= 0 || (thresholds && counts), MCBA_ERR_ARG, "null thresholds or counts");
    REQUIRE(ctx->table && ctx->errors_current, MCBA_ERR_STATE, "mcba_table_errors has not run since the parameters or the selection changed");
    REQUIRE(which == MCBA_TABLE_VALID || which == MCBA_TABLE_INLIERS, MCBA_ERR_ARG, "unknown table selection");
    if (n <= 0) return;
    const int64_t count = which == MCBA_TABLE_VALID ? ctx->n_valid : ctx->n_inliers;
    CK(ctx->table_out.alloc((size_t)n)); CK(ctx->table_ranks.alloc((size_t)n));
    CK(cudaMemcpyAsync(ctx->table_out.p, thresholds, sizeof(double) * n, cudaMemcpyHostToDevice, ctx->stream));
    k_count_below<<<(n + 127) / 128, 128, 0, ctx->stream>>>(which == MCBA_TABLE_VALID ? ctx->err_sorted.p : ctx->err_inl_sorted.p, count,
                                                          ctx->table_out.p, n, ctx->table_ranks.p); CKL();
    CK(cudaMemcpyAsync(counts, ctx->table_ranks.p, sizeof(int64_t) * n, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
  });
}

int mcba_table_reject(mcba_ctx* ctx, double threshold, int64_t* n_valid, int64_t* n_keep) {
  return api(ctx, [&] {
    REQUIRE(ctx->table && ctx->errors_current && ctx->table_selected == MCBA_TABLE_VALID, MCBA_ERR_STATE,
            "mcba_table_errors has not run since the parameters or the selection changed");
    const DeviceProblem& P = ctx->P;
    cudaStream_t s = ctx->stream;
    const size_t dense = table_dense(ctx);
    double kept = 0.0;
    if (dense) CK(cudaMemsetAsync(ctx->inlier_mask.p, 0, dense, s));
    if (P.N > 0) {
      const int blocks = std::max(1, std::min((P.V + TABLE_WARPS - 1) / TABLE_WARPS, ctx->num_sms * 8));
      k_table_reject<<<blocks, TABLE_WARPS * 32, 0, s>>>(P, ctx->err_valid.p, threshold, ctx->inlier_mask.p, ctx->table_part.p); CKL();
      double* d_sum = ctx->table_part.p + (size_t)3 * P.V;
      k_sum_partials<<<1, 1024, 0, s>>>(ctx->table_part.p, P.V, 1, 1, d_sum); CKL();
      CK(cudaMemcpyAsync(&kept, d_sum, sizeof(double), cudaMemcpyDeviceToHost, s));
    }
    CK(cudaStreamSynchronize(s));
    ctx->n_inliers = (int64_t)llround(kept);
    ctx->errors_current = false;           // the sorted inlier errors describe the previous mask
    if (n_valid) *n_valid = P.N;
    if (n_keep) *n_keep = ctx->n_inliers;
  });
}

int mcba_set_params(mcba_ctx* ctx, const double* cam_rt, const double* board_rt, const double* frame_rt, const double* intrinsics) {
  return api(ctx, [&] {
    REQUIRE(ctx->uploaded, MCBA_ERR_STATE, "no problem uploaded");
    REQUIRE(cam_rt && board_rt && intrinsics && (frame_rt || ctx->P.F == 0 || ctx->P.fb == 0), MCBA_ERR_ARG, "null parameter array");
    const DeviceProblem& P = ctx->P;
    ctx->errors_current = false;
    CK(cudaMemcpyAsync(P.cam_rt, cam_rt, sizeof(double) * P.C * 6, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(P.board_rt, board_rt, sizeof(double) * P.B * 6, cudaMemcpyHostToDevice, ctx->stream));
    if (P.F && P.fb) CK(cudaMemcpyAsync(P.frame_rt, frame_rt, sizeof(double) * P.F * P.fb, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(P.intr, intrinsics, sizeof(double) * P.C * P.kint, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
  });
}

// Same state as 4x4 pose matrices (PoseSet.poses): the rotation-vector conversions of transform/rtvec.py run on the device.
// mats: f64[C+B+F][4][4] in the order cameras, boards, frames.
int mcba_set_state_matrices(mcba_ctx* ctx, const double* mats, const double* intrinsics) {
  return api(ctx, [&] {
    REQUIRE(ctx->uploaded, MCBA_ERR_STATE, "no problem uploaded");
    REQUIRE(mats && intrinsics, MCBA_ERR_ARG, "null parameter array");
    const DeviceProblem& P = ctx->P;
    const int np = P.C + P.B + P.F;
    ctx->errors_current = false;
    CK(ctx->pose_mats.alloc((size_t)np * 16));
    CK(cudaMemcpyAsync(ctx->pose_mats.p, mats, sizeof(double) * 16 * np, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(P.intr, intrinsics, sizeof(double) * P.C * P.kint, cudaMemcpyHostToDevice, ctx->stream));
    k_matrices_to_state<<<(np + 127) / 128, 128, 0, ctx->stream>>>(P.C, P.B, P.F, ctx->pose_mats.p, P.cam_rt, P.board_rt, P.frame_rt, P.fb); CKL();
    CK(cudaStreamSynchronize(ctx->stream));     // the host arrays are borrowed only for the call
  });
}

int mcba_get_state_matrices(mcba_ctx* ctx, double* mats, double* intrinsics) {
  return api(ctx, [&] {
    REQUIRE(ctx->uploaded, MCBA_ERR_STATE, "no problem uploaded");
    const DeviceProblem& P = ctx->P;
    const int np = P.C + P.B + P.F;
    if (mats) {
      CK(ctx->pose_mats.alloc((size_t)np * 16));
      const PoseT* derived = nullptr;
      if (P.motion == MOTION_HAND_EYE) { prepare(ctx, with_state(ctx, false)); derived = P.frame_T; }
      k_state_to_matrices<<<(np + 127) / 128, 128, 0, ctx->stream>>>(P.C, P.B, P.F, P.cam_rt, P.board_rt, P.frame_rt, ctx->pose_mats.p, P.fb, derived); CKL();
      CK(cudaMemcpyAsync(mats, ctx->pose_mats.p, sizeof(double) * 16 * np, cudaMemcpyDeviceToHost, ctx->stream));
    }
    if (intrinsics) CK(cudaMemcpyAsync(intrinsics, P.intr, sizeof(double) * P.C * P.kint, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
  });
}

// RollingFrames (motion/rolling_frames.py:66-150): the frames of mcba_set_state_matrices are the start poses; the end poses
// f64[F][4][4] and the image heights f64[C] that turn an observed row into the blend weight (rolling_times, 15-19) come here.
int mcba_set_rolling(mcba_ctx* ctx, const double* end_pose_matrices, const double* image_heights) {
  return api(ctx, [&] {
    REQUIRE(ctx->uploaded, MCBA_ERR_STATE, "no problem uploaded");
    const DeviceProblem& P = ctx->P;
    REQUIRE(P.motion == MOTION_ROLLING, MCBA_ERR_STATE, "the problem was not uploaded with MCBA_MOTION_ROLLING");
    REQUIRE((end_pose_matrices || P.F == 0) && image_heights, MCBA_ERR_ARG, "null parameter array");
    for (int c = 0; c < P.C; c++) REQUIRE(image_heights[c] > 0, MCBA_ERR_ARG, "image heights must be positive");
    ctx->errors_current = false;
    CK(cudaMemcpyAsync(ctx->img_h.p, image_heights, sizeof(double) * P.C, cudaMemcpyHostToDevice, ctx->stream));
    if (P.F) {
      CK(ctx->pose_mats.alloc((size_t)P.F * 16));
      CK(cudaMemcpyAsync(ctx->pose_mats.p, end_pose_matrices, sizeof(double) * 16 * P.F, cudaMemcpyHostToDevice, ctx->stream));
      // "cameras = 0, boards = 0, frames = F" view of the same kernel, writing the second half of every frame block
      k_matrices_to_state<<<(P.F + 127) / 128, 128, 0, ctx->stream>>>(0, 0, P.F, ctx->pose_mats.p, nullptr, nullptr, P.frame_rt + 6, 12); CKL();
    }
    CK(cudaStreamSynchronize(ctx->stream));
  });
}

int mcba_get_rolling(mcba_ctx* ctx, double* end_pose_matrices) {
  return api(ctx, [&] {
    REQUIRE(end_pose_matrices, MCBA_ERR_ARG, "null parameter array");
    REQUIRE(ctx->uploaded, MCBA_ERR_STATE, "no problem uploaded");
    const DeviceProblem& P = ctx->P;
    REQUIRE(P.motion == MOTION_ROLLING, MCBA_ERR_STATE, "the problem was not uploaded with MCBA_MOTION_ROLLING");
    if (P.F) {
      CK(ctx->pose_mats.alloc((size_t)P.F * 16));
      k_state_to_matrices<<<(P.F + 127) / 128, 128, 0, ctx->stream>>>(0, 0, P.F, nullptr, nullptr, P.frame_rt + 6, ctx->pose_mats.p, 12, nullptr); CKL();
      CK(cudaMemcpyAsync(end_pose_matrices, ctx->pose_mats.p, sizeof(double) * 16 * P.F, cudaMemcpyDeviceToHost, ctx->stream));
    }
    CK(cudaStreamSynchronize(ctx->stream));
  });
}

// HandEye (motion/hand_eye.py:14-90): frame pose f = gripper_wrt_camera base_wrt_gripper[f] world_wrt_base; the arm poses are
// constants, the two outer transforms are the 12 motion parameters.  The frames of mcba_set_state_matrices are ignored.
int mcba_set_hand_eye(mcba_ctx* ctx, const double* base_wrt_gripper, const double* world_wrt_base, const double* gripper_wrt_camera) {
  return api(ctx, [&] {
    REQUIRE(ctx->uploaded, MCBA_ERR_STATE, "no problem uploaded");
    const DeviceProblem& P = ctx->P;
    REQUIRE(P.motion == MOTION_HAND_EYE, MCBA_ERR_STATE, "the problem was not uploaded with MCBA_MOTION_HAND_EYE");
    REQUIRE((base_wrt_gripper || P.F == 0) && world_wrt_base && gripper_wrt_camera, MCBA_ERR_ARG, "null parameter array");
    ctx->errors_current = false;
    std::vector<PoseT> arms((size_t)std::max(P.F, 1));
    for (int f = 0; f < P.F; f++) {
      const double* M = base_wrt_gripper + (size_t)16 * f;
      PoseT t{};
      for (int r = 0; r < 3; r++) { t.R[3 * r] = M[4 * r]; t.R[3 * r + 1] = M[4 * r + 1]; t.R[3 * r + 2] = M[4 * r + 2]; t.t[r] = M[4 * r + 3]; }
      arms[(size_t)f] = t;
    }
    CK(cudaMemcpyAsync(ctx->arm_T.p, arms.data(), sizeof(PoseT) * arms.size(), cudaMemcpyHostToDevice, ctx->stream));
    CK(ctx->pose_mats.alloc(32));
    CK(cudaMemcpyAsync(ctx->pose_mats.p, world_wrt_base, sizeof(double) * 16, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(ctx->pose_mats.p + 16, gripper_wrt_camera, sizeof(double) * 16, cudaMemcpyHostToDevice, ctx->stream));
    k_matrices_to_state<<<1, 128, 0, ctx->stream>>>(0, 0, 2, ctx->pose_mats.p, nullptr, nullptr, P.he_rt, 6); CKL();
    CK(cudaStreamSynchronize(ctx->stream));
  });
}

int mcba_get_hand_eye(mcba_ctx* ctx, double* world_wrt_base, double* gripper_wrt_camera) {
  return api(ctx, [&] {
    REQUIRE(ctx->uploaded, MCBA_ERR_STATE, "no problem uploaded");
    const DeviceProblem& P = ctx->P;
    REQUIRE(P.motion == MOTION_HAND_EYE, MCBA_ERR_STATE, "the problem was not uploaded with MCBA_MOTION_HAND_EYE");
    CK(ctx->pose_mats.alloc(32));
    k_state_to_matrices<<<1, 128, 0, ctx->stream>>>(0, 0, 2, nullptr, nullptr, P.he_rt, ctx->pose_mats.p, 6, nullptr); CKL();
    if (world_wrt_base) CK(cudaMemcpyAsync(world_wrt_base, ctx->pose_mats.p, sizeof(double) * 16, cudaMemcpyDeviceToHost, ctx->stream));
    if (gripper_wrt_camera) CK(cudaMemcpyAsync(gripper_wrt_camera, ctx->pose_mats.p + 16, sizeof(double) * 16, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
  });
}

// OpenCV's CALIB_FIX_* flags: intrinsic parameters held at their current values.  The mask lives in the problem descriptor that every
// launch takes by value (and so in the key of the solve's cached graph); setup_problem clears it on every upload.
int mcba_set_fixed_intrinsics(mcba_ctx* ctx, const uint8_t* fixed) {
  return api(ctx, [&] {
    REQUIRE(ctx->uploaded, MCBA_ERR_STATE, "no problem uploaded");
    DeviceProblem& P = ctx->P;
    uint32_t m = 0;
    for (int i = 0; fixed && i < P.kint; i++) {
      REQUIRE(fixed[i] <= 1, MCBA_ERR_ARG, "fixed intrinsics: every entry must be 0 or 1");
      if (fixed[i]) m |= 1u << i;
    }
    REQUIRE(!P.fix_aspect || (m & 1u) == ((m >> 1) & 1u), MCBA_ERR_ARG,
            "fixed intrinsics: under MCBA_OPT_FIX_ASPECT fy follows fx, so fx and fy are fixed together or not at all");
    P.fixed_intr = m;
  });
}

// scipy's tr_solver: like the fixed-intrinsics mask a field of the problem descriptor (graph key; cleared by every upload)
int mcba_set_trust_region(mcba_ctx* ctx, int32_t mode) {
  return api(ctx, [&] {
    REQUIRE(ctx->uploaded, MCBA_ERR_STATE, "no problem uploaded");
    REQUIRE(mode == MCBA_TR_SUBSPACE || mode == MCBA_TR_EXACT, MCBA_ERR_ARG, "trust region: MCBA_TR_SUBSPACE or MCBA_TR_EXACT");
    ctx->P.tr_exact = mode == MCBA_TR_EXACT ? 1 : 0;
  });
}

int mcba_last_alpha_iterations(mcba_ctx* ctx, int32_t* total) {
  return api(ctx, [&] {
    REQUIRE(total, MCBA_ERR_ARG, "null argument");
    *total = ctx->last_alpha_iters;
  });
}

int mcba_get_params(mcba_ctx* ctx, double* cam_rt, double* board_rt, double* frame_rt, double* intrinsics) {
  return api(ctx, [&] {
    REQUIRE(ctx->uploaded, MCBA_ERR_STATE, "no problem uploaded");
    const DeviceProblem& P = ctx->P;
    if (cam_rt) CK(cudaMemcpyAsync(cam_rt, P.cam_rt, sizeof(double) * P.C * 6, cudaMemcpyDeviceToHost, ctx->stream));
    if (board_rt) CK(cudaMemcpyAsync(board_rt, P.board_rt, sizeof(double) * P.B * 6, cudaMemcpyDeviceToHost, ctx->stream));
    if (frame_rt && P.F && P.fb) CK(cudaMemcpyAsync(frame_rt, P.frame_rt, sizeof(double) * P.F * P.fb, cudaMemcpyDeviceToHost, ctx->stream));
    if (intrinsics) CK(cudaMemcpyAsync(intrinsics, P.intr, sizeof(double) * P.C * P.kint, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
  });
}

int mcba_num_params(mcba_ctx* ctx, int64_t* n) {
  return api(ctx, [&] {
    REQUIRE(n, MCBA_ERR_ARG, "null argument");
    REQUIRE(ctx->uploaded, MCBA_ERR_STATE, "no problem uploaded");
    *n = ctx->P.n;
  });
}

static void read_x_canonical(mcba_ctx* ctx, double* x) {
  const DeviceProblem& P = ctx->P;
  if (P.n == 0) return;
  k_gather_params<<<(P.n + 255) / 256, 256, 0, ctx->stream>>>(P, ctx->x.p, P.cam_rt, P.board_rt, P.frame_rt, P.intr); CKL();
  std::vector<double> h((size_t)P.n);
  CK(cudaMemcpyAsync(h.data(), ctx->x.p, sizeof(double) * P.n, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  for (int i = 0; i < P.n; i++) x[ctx->perm[(size_t)i]] = h[(size_t)i];
}
static void write_x_canonical(mcba_ctx* ctx, const double* x, double* dev_x) {
  const DeviceProblem& P = ctx->P;
  if (P.n == 0) return;
  std::vector<double> h((size_t)P.n);
  for (int i = 0; i < P.n; i++) h[(size_t)i] = x[ctx->perm[(size_t)i]];
  CK(cudaMemcpyAsync(dev_x, h.data(), sizeof(double) * P.n, cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
}
// the current state := x (canonical order)
static void set_param_vec(mcba_ctx* ctx, const double* x) {
  ctx->errors_current = false;
  write_x_canonical(ctx, x, ctx->x.p);
  set_state_from_x(ctx, ctx->x.p, false);
  CK(cudaStreamSynchronize(ctx->stream));
}

int mcba_get_param_vec(mcba_ctx* ctx, double* x) {
  return api(ctx, [&] {
    REQUIRE(x, MCBA_ERR_ARG, "null parameter vector");
    REQUIRE(ctx->uploaded, MCBA_ERR_STATE, "no problem uploaded");
    read_x_canonical(ctx, x);
  });
}

int mcba_set_param_vec(mcba_ctx* ctx, const double* x) {
  return api(ctx, [&] {
    REQUIRE(x, MCBA_ERR_ARG, "null parameter vector");
    REQUIRE(ctx->uploaded, MCBA_ERR_STATE, "no problem uploaded");
    set_param_vec(ctx, x);
  });
}

int mcba_residuals(mcba_ctx* ctx, const double* x, double* r_out, double* cost) {
  return api(ctx, [&] {
    REQUIRE(ctx->uploaded, MCBA_ERR_STATE, "no problem uploaded");
    bool trial = false;
    if (x) {
      // evaluate at x without disturbing the stored parameters: trial state = current state overwritten by x
      write_x_canonical(ctx, x, ctx->x_new.p);
      set_state_from_x(ctx, ctx->x_new.p, true);
      trial = true;
    } else {
      prepare(ctx, with_state(ctx, false));
    }
    DeviceProblem P = with_state(ctx, trial);
    if (r_out && P.N > 0) {
      DevBuf<double> dr; CK(dr.alloc((size_t)2 * P.N));
      ViewKernelArgs a{}; a.resid = dr.p;
      launch_views<MODE_RESID>(ctx, P, a);
      CK(cudaMemcpyAsync(r_out, dr.p, sizeof(double) * 2 * P.N, cudaMemcpyDeviceToHost, ctx->stream));
      CK(cudaStreamSynchronize(ctx->stream));
    }
    if (cost) {
      trial_cost(ctx, 0, 1.0, trial);
      CK(cudaMemcpyAsync(cost, ctx->eval_cost.p, sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
      CK(cudaStreamSynchronize(ctx->stream));
    }
  });
}

int mcba_reprojection_error(mcba_ctx* ctx, double* err) {
  return api(ctx, [&] {
    REQUIRE(err, MCBA_ERR_ARG, "null argument");
    REQUIRE(ctx->uploaded, MCBA_ERR_STATE, "no problem uploaded");
    DeviceProblem P = with_state(ctx, false);
    if (P.N == 0) return;
    prepare(ctx, P);
    DevBuf<double> de; CK(de.alloc((size_t)P.N));
    ViewKernelArgs a{}; a.err = de.p;
    launch_views<MODE_ERROR>(ctx, P, a);
    CK(cudaMemcpyAsync(err, de.p, sizeof(double) * P.N, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
  });
}

int mcba_linearize(mcba_ctx* ctx, const double* x, double* JtJ, double* Jtr, double* cost) {
  return api(ctx, [&] {
    REQUIRE(ctx->uploaded, MCBA_ERR_STATE, "no problem uploaded");
    const DeviceProblem& P = ctx->P;
    if (x) set_param_vec(ctx, x);
    else prepare(ctx, with_state(ctx, false));
    linearize(ctx, 0, 1.0);
    const int n = P.n, n_s = P.n_s, F = P.motion_on ? P.F : 0;
    const int fb = P.fb;
    std::vector<double> hHss((size_t)n_s * n_s), hg((size_t)n), hHff((size_t)F * fb * fb), hW((size_t)F * n_s * fb);
    if (n_s) CK(cudaMemcpyAsync(hHss.data(), ctx->Hss.p, sizeof(double) * hHss.size(), cudaMemcpyDeviceToHost, ctx->stream));
    if (n) CK(cudaMemcpyAsync(hg.data(), ctx->g.p, sizeof(double) * n, cudaMemcpyDeviceToHost, ctx->stream));
    if (F) CK(cudaMemcpyAsync(hHff.data(), ctx->Hff.p, sizeof(double) * hHff.size(), cudaMemcpyDeviceToHost, ctx->stream));
    if (F && n_s) CK(cudaMemcpyAsync(hW.data(), ctx->W.p, sizeof(double) * hW.size(), cudaMemcpyDeviceToHost, ctx->stream));
    double hcost = 0;
    CK(cudaMemcpyAsync(&hcost, ctx->lin_cost.p, sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    const std::vector<int>& pm = ctx->perm;
    if (JtJ) {
      std::fill(JtJ, JtJ + (size_t)n * n, 0.0);
      for (int i = 0; i < n_s; i++) for (int j = 0; j < n_s; j++) JtJ[(size_t)pm[i] * n + pm[j]] = hHss[(size_t)i * n_s + j];
      for (int f = 0; f < F; f++) {
        for (int i = 0; i < fb; i++) for (int j = 0; j < fb; j++) JtJ[(size_t)pm[n_s + fb * f + i] * n + pm[n_s + fb * f + j]] = hHff[((size_t)f * fb + i) * fb + j];
        for (int s = 0; s < n_s; s++) for (int j = 0; j < fb; j++) {
          const double w = hW[((size_t)f * n_s + s) * fb + j];
          JtJ[(size_t)pm[s] * n + pm[n_s + fb * f + j]] = w;
          JtJ[(size_t)pm[n_s + fb * f + j] * n + pm[s]] = w;
        }
      }
    }
    if (Jtr) for (int i = 0; i < n; i++) Jtr[pm[i]] = hg[(size_t)i];
    if (cost) *cost = hcost;
  });
}

int mcba_solve(mcba_ctx* ctx, const mcba_solve_opts* opts, mcba_solve_result* result, mcba_log_row* log, int32_t log_capacity) {
  return api(ctx, [&] {
    REQUIRE(opts && result, MCBA_ERR_ARG, "null options or result");
    REQUIRE(ctx->uploaded, MCBA_ERR_STATE, "no problem uploaded");
    REQUIRE(opts->loss >= 0 && opts->loss <= 4, MCBA_ERR_ARG, "unknown loss");
    REQUIRE(opts->max_nfev > 0, MCBA_ERR_ARG, "max_nfev must be positive");
    REQUIRE(opts->f_scale > 0, MCBA_ERR_ARG, "f_scale must be positive");
    REQUIRE(ctx->world == 1 || !ctx->P.tr_exact, MCBA_ERR_UNSUPPORTED,
            "tr_solver='exact' on several ranks: the alpha search would exchange the reduced system once per alpha");
    REQUIRE(ctx->world == 1 || ctx->peer_ready, MCBA_ERR_STATE, "several ranks: the exchanges run over NVLink peer memory (mcba_peer_export / mcba_peer_import first)");
    const DeviceProblem& P = ctx->P;
    REQUIRE(ctx->world == 1 || (size_t)P.n_s * P.n_s + 2 * (size_t)P.n_s + 16 <= (size_t)ctx->peer_cap, MCBA_ERR_STATE,
            "the reduced normal equations do not fit the NVLink exchange slots: export larger peer buffers (mcba_peer_export cap >= n_s^2 + 2 n_s + 16)");
    cudaStream_t s = ctx->stream;
    const int n = P.n;
    memset(result, 0, sizeof(*result));
    ctx->launches = 0;
    ctx->last_alpha_iters = 0;
    ctx->errors_current = false;
    struct EventPair {       // destroyed on every return path
      cudaEvent_t a = nullptr, b = nullptr;
      ~EventPair() { if (a) cudaEventDestroy(a); if (b) cudaEventDestroy(b); }
    } ev;
    CK(cudaEventCreate(&ev.a)); CK(cudaEventCreate(&ev.b));
    CK(cudaEventRecord(ev.a, s));

    SolverState h{};
    h.ftol = opts->ftol; h.xtol = opts->xtol; h.gtol = opts->gtol; h.reg_floor = 1e-12; h.max_nfev = opts->max_nfev;
    h.nfev = 1; h.njev = 1; h.iteration = 0; h.status = -99; h.first_scale = 1;
    if (n == 0) {      // nothing to optimise: report the cost and leave
      prepare(ctx, with_state(ctx, false));
      linearize(ctx, opts->loss, opts->f_scale);
      // one number: the host's collective is the simplest exchange (no solver state involved)
      REQUIRE(ctx->world == 1, MCBA_ERR_UNSUPPORTED, "nothing to optimise on several ranks: sum mcba_residuals' cost on the host");
      CK(cudaMemcpyAsync(&h.cost, ctx->lin_cost.p, sizeof(double), cudaMemcpyDeviceToHost, s));
      CK(cudaStreamSynchronize(s));
      result->initial_cost = h.cost; result->cost = h.cost; result->nfev = 1; result->njev = 1; result->status = 1;
      if (log && log_capacity > 0) { log[0] = mcba_log_row{0, 1, h.cost, NAN, NAN, 0.0}; result->n_log = 1; }
      CK(cudaEventRecord(ev.b, s)); CK(cudaEventSynchronize(ev.b));
      float ms0 = 0; cudaEventElapsedTime(&ms0, ev.a, ev.b);
      result->device_ms = ms0; result->kernel_launches = ctx->launches;
      return;
    }
    CK(cudaMemcpyAsync(ctx->state.p, &h, sizeof(h), cudaMemcpyHostToDevice, s));
    // x0 and the trial state := the current state; its pose tables
    k_gather_params<<<(n + 255) / 256, 256, 0, s>>>(P, ctx->x.p, P.cam_rt, P.board_rt, P.frame_rt, P.intr); CKL();
    CK(cudaMemcpyAsync(ctx->x_new.p, ctx->x.p, sizeof(double) * n, cudaMemcpyDeviceToDevice, s));
    copy_state_to_trial(ctx);
    prepare(ctx, with_state(ctx, true));
    const int cap = std::max(8, opts->max_nfev + 4);
    CK(ctx->dev_log.alloc((size_t)cap));

    run_lm_loop(ctx, opts->loss, opts->f_scale, cap);

    CK(cudaMemcpyAsync(&h, ctx->state.p, sizeof(h), cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    REQUIRE(h.status != -2, MCBA_ERR_NONFINITE, "Residuals are not finite in the initial point.");
    REQUIRE(h.status != -3, MCBA_ERR_NCCL, "a peer rank did not answer an in-kernel exchange (timeout): the ranks left mcba_solve out of step");
    const int nlog = std::min(h.nlog, cap);
    std::vector<mcba_log_row> rows((size_t)std::max(nlog, 1));
    if (nlog > 0) CK(cudaMemcpyAsync(rows.data(), ctx->dev_log.p, sizeof(mcba_log_row) * nlog, cudaMemcpyDeviceToHost, s));
    // leave the context consistent: pose tables of the final (current) state
    prepare(ctx, with_state(ctx, false));
    CK(cudaEventRecord(ev.b, s));
    CK(cudaEventSynchronize(ev.b));
    float ms = 0; cudaEventElapsedTime(&ms, ev.a, ev.b);
    if (nlog > 0) result->initial_cost = rows[0].cost;
    if (log) for (int i = 0; i < nlog && i < log_capacity; i++) log[i] = rows[(size_t)i];
    result->cost = h.cost; result->optimality = h.g_norm; result->nfev = h.nfev; result->njev = h.njev;
    result->status = h.status == -99 ? 0 : h.status; result->n_log = std::min(nlog, (int)log_capacity); result->device_ms = ms;
    if (ctx->graph_launched) ctx->launches += ctx->sg.body_launches * (h.nfev + h.relins);      // the WHILE node ran the body once per evaluation and relinearisation
    ctx->last_alpha_iters = h.alpha_iters;
    result->kernel_launches = ctx->launches; result->chol_retries = h.chol_fail;
  });
}

int mcba_bench_info(mcba_ctx* ctx, int which, int64_t* corners, int64_t* bytes, int32_t* launches) {
  return api(ctx, [&] {
    REQUIRE(ctx->uploaded, MCBA_ERR_STATE, "no problem uploaded");
    const DeviceProblem& P = ctx->P;
    int64_t per_corner = 18, per_view = 16, l = 1;
    if (which == MCBA_BENCH_RESIDUAL) per_corner = 18 + 4 + 16;
    if (corners) *corners = P.N;
    if (bytes) *bytes = per_corner * P.N + per_view * P.V;      // per launch
    if (launches) *launches = (int32_t)l;
  });
}

int mcba_bench_launch(mcba_ctx* ctx, int which, int repeats) {
  return api(ctx, [&] {
    REQUIRE(ctx->uploaded, MCBA_ERR_STATE, "no problem uploaded");
    DeviceProblem P = with_state(ctx, false);
    if (!(which & MCBA_BENCH_NO_PREPARE)) prepare(ctx, P);
    which &= ~MCBA_BENCH_NO_PREPARE;
    for (int i = 0; i < repeats; i++) {
      ViewKernelArgs a{}; a.loss = 0; a.f_scale = 1.0;
      if (which == MCBA_BENCH_LINEARIZE) launch_linearize(ctx, P, 0, 1.0);
      else if (which == MCBA_BENCH_COST) { a.view_cost = ctx->view_cost.p; launch_views<MODE_COST>(ctx, P, a); }
      else throw Failure{MCBA_ERR_ARG, "unsupported bench kernel"};
    }
  });
}

}  // extern "C"
