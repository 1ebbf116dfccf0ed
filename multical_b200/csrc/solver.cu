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
#include <type_traits>
#include <vector>

#include "../../include/mcba.h"
#include "solver_kernels.cuh"
#include "linearize.cuh"
#include "lm_kernel.cuh"
#include "pack_kernels.cuh"
#include "table_kernels.cuh"
#include "pnp_kernels.cuh"
#include "intrinsics_kernels.cuh"

using namespace mcba;

namespace {

thread_local std::string g_create_error;

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

}  // namespace

struct mcba_ctx {
  int device = 0;
  cudaStream_t stream = nullptr;       // the stream every entry point works on
  cudaStream_t own_stream = nullptr;   // created by mcba_create; `stream` differs after mcba_set_stream
  std::string err;
  int rank = 0, world = 1;
  int launches = 0;
  int num_sms = 132;

  bool uploaded = false;
  DeviceProblem P{};
  // problem arrays
  DevBuf<double2> obs; DevBuf<uint16_t> pid; DevBuf<uint32_t> orig;
  DevBuf<int> view_start, view_cam, view_frame, view_board, frame_view_start;
  DevBuf<uint8_t> dense_mask, view_valid; DevBuf<double2> dense_pts; DevBuf<float2> dense_pts32; DevBuf<int> scan;
  cudaStream_t copy_stream = nullptr; cudaEvent_t copy_done = nullptr, copy_go = nullptr;      // observations of mcba_upload_dense* in flight beside the view count
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
  DevBuf<double> x, x_new, sinv, d, gh, gn, Y, Lf, zf, S, rhs, Linv;
  DevBuf<double> lin_cost, eval_cost;     // cost at the last linearisation (k_reduce_shared), cost of mcba_residuals
  DevBuf<SolverState> state;
  // NVLink peer-memory exchange of the solver kernel (lm_kernel.cuh LmPeer)
  double* peer_own = nullptr; int peer_cap = 0; bool peer_ready = false;
  double* peer_base[PEER_MAX_WORLD] = {nullptr};
  std::vector<void*> peer_opened;
  std::vector<int> perm;   // internal index -> canonical param_vec index
  // resident point table (mcba_table_*): `valid` and inlier masks, sorted per-corner errors
  bool table = false; int table_selected = -1; bool errors_current = false;
  mcba_problem_desc table_desc{};
  int64_t n_valid = 0, n_inliers = 0;
  DevBuf<uint8_t> valid_mask, inlier_mask;
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
};

#define CK(call)                                                                                   \
  do {                                                                                             \
    cudaError_t e_ = (call);                                                                       \
    if (e_ != cudaSuccess) {                                                                       \
      ctx->err = std::string(#call) + ": " + cudaGetErrorString(e_);                               \
      return MCBA_ERR_CUDA;                                                                        \
    }                                                                                              \
  } while (0)
#define CKL()                                                                                      \
  do {                                                                                             \
    ctx->launches++;                                                                               \
    cudaError_t e_ = cudaGetLastError();                                                           \
    if (e_ != cudaSuccess) { ctx->err = std::string("kernel launch: ") + cudaGetErrorString(e_); return MCBA_ERR_CUDA; } \
  } while (0)
#define REQUIRE(cond, code, msg)                                                                   \
  do { if (!(cond)) { ctx->err = msg; return code; } } while (0)

namespace {

// parameters of block-structured vector x (internal order) <-> full parameter state
__global__ void k_scatter_params(DeviceProblem p, const double* x, double* cam_rt, double* board_rt, double* frame_rt, double* intr) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= p.n) return;
  const double v = x[i];
  if (i >= p.n_s) { frame_rt[i - p.n_s] = v; return; }
  if (p.off_cp >= 0 && i >= p.off_cp && i < p.off_cp + 6 * p.C) { cam_rt[i - p.off_cp] = v; return; }
  if (p.off_bp >= 0 && i >= p.off_bp && i < p.off_bp + 6 * p.B) { board_rt[i - p.off_bp] = v; return; }
  if (p.off_in >= 0 && i >= p.off_in && i < p.off_in + p.kint * p.C) { intr[i - p.off_in] = v; return; }
  if (p.off_pt >= 0 && i >= p.off_pt && i < p.off_pt + 3 * p.B * p.P) { p.board_pts[i - p.off_pt] = v; return; }
  if (p.off_he >= 0 && i >= p.off_he && i < p.off_he + 12) p.he_rt[i - p.off_he] = v;
}
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
// copies the fixed blocks so that a trial state is complete; with fix_aspect fy follows fx (camera.py:159-160)
__global__ void k_fix_aspect(DeviceProblem p, double* intr) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c < p.C && p.fix_aspect) intr[c * p.kint + 1] = intr[c * p.kint];
}

template <int MODE>
int launch_views(mcba_ctx* ctx, const DeviceProblem& P, const ViewKernelArgs& a) {
  const int blocks = std::max(1, std::min((P.V + VIEW_WARPS - 1) / VIEW_WARPS, ctx->num_sms * 8));
  const int th = VIEW_WARPS * 32;
  cudaStream_t s = ctx->stream;
  with_model(P.model, P.motion == MOTION_ROLLING, [&](auto M, auto R) {
    constexpr int MODEL = decltype(M)::value; constexpr bool ROLL = decltype(R)::value;
    k_views<MODEL, MODE, ROLL><<<blocks, th, 0, s>>>(P, a);
  });
  CKL();
  return MCBA_OK;
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
int launch_linearize(mcba_ctx* ctx, const DeviceProblem& P, int loss, double f_scale) {
  if (P.F == 0) return MCBA_OK;
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
  return MCBA_OK;
}
// per-CTA records -> H_ss, g_s, cost (stores, fixed summation order)
int launch_reduce_shared(mcba_ctx* ctx, const DeviceProblem& P) {
  ReduceArgs r{}; r.spart = ctx->spart.p; r.nparts = P.F > 0 ? ctx->lin_grid : 0; r.Hss = ctx->Hss.p; r.g = ctx->g.p; r.bpart = ctx->bpart.p;
  r.frame_cost = ctx->frame_cost.p; r.F = P.F; r.cost_out = ctx->lin_cost.p; r.cam_counter = ctx->cam_counter.p; r.sred = ctx->sred.p;
  const size_t sm = sizeof(double) * reduce_smem_doubles(P.T, P.D, P.B);
  const int grid = P.C * reduce_slices(lin_record_doubles(P.T, P.D, P.B));
  if (P.motion == MOTION_ROLLING) k_reduce_shared<2><<<grid, RED_THREADS, sm, ctx->stream>>>(P, r);
  else k_reduce_shared<1><<<grid, RED_THREADS, sm, ctx->stream>>>(P, r);
  CKL();
  return MCBA_OK;
}

// DeviceProblem view whose parameter pointers are the trial state
DeviceProblem with_state(const mcba_ctx* ctx, bool trial) {
  DeviceProblem P = ctx->P;
  if (trial) set_state_pointers(P, ctx->trial.p, ctx->layout);
  return P;
}

int prepare(mcba_ctx* ctx, const DeviceProblem& P) {
  const int np = P.C + P.B + P.F * P.npf + (P.motion == MOTION_HAND_EYE ? 2 : 0);
  k_prepare<<<(np + 127) / 128, 128, 0, ctx->stream>>>(P, P.cam_rt, P.board_rt, P.frame_rt);
  CKL();
  return MCBA_OK;
}

// push vector x (internal order) into the (trial or current) parameter state and rebuild the pose tables
int set_state_from_x(mcba_ctx* ctx, const double* x, bool trial) {
  DeviceProblem P = with_state(ctx, trial);
  if (P.n > 0) {
    k_scatter_params<<<(P.n + 255) / 256, 256, 0, ctx->stream>>>(P, x, P.cam_rt, P.board_rt, P.frame_rt, P.intr);
    CKL();
    if (P.fix_aspect && P.off_in >= 0) { k_fix_aspect<<<(P.C + 127) / 128, 128, 0, ctx->stream>>>(P, P.intr); CKL(); }
  }
  return prepare(ctx, P);
}

// The normal equations and the cost at the (trial or current) state, whose pose tables must already describe it: k_linearize, its per-CTA
// records -> H_ss, g_s, cost (k_reduce_shared), then boards=True: the board-point blocks on top (k_point_blocks), then hand-eye: the
// hand-eye rows and columns from the frame blocks (k_fold_hand_eye, last: it reads the point rows of W_f)
int linearize(mcba_ctx* ctx, int loss, double f_scale, bool trial = false) {
  DeviceProblem P = with_state(ctx, trial);
  cudaStream_t s = ctx->stream;
  int r = launch_linearize(ctx, P, loss, f_scale); if (r) return r;
  if (P.off_pt >= 0) {         // k_point_blocks adds the point rows / columns (atomics): they start at zero
    CK(cudaMemsetAsync(ctx->Hss.p, 0, sizeof(double) * (size_t)P.n_s * P.n_s, s));
    CK(cudaMemsetAsync(ctx->g.p, 0, sizeof(double) * (size_t)std::max(P.n_s, 1), s));
  }
  r = launch_reduce_shared(ctx, P); if (r) return r;
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
  return MCBA_OK;
}

// cost at the (trial or current) state -> eval_cost
int trial_cost(mcba_ctx* ctx, int loss, double f_scale, bool trial) {
  DeviceProblem P = with_state(ctx, trial);
  ViewKernelArgs a{}; a.loss = loss; a.f_scale = f_scale; a.view_cost = ctx->view_cost.p;
  int r = launch_views<MODE_COST>(ctx, P, a); if (r) return r;
  k_sum_partials<<<1, 1024, 0, ctx->stream>>>(ctx->view_cost.p, P.V, 1, 1, ctx->eval_cost.p); CKL();
  return MCBA_OK;
}

// ---------------------------------------------------------------- the device-resident trust-region loop (lm_kernel.cuh)
// trial parameter state := current state
int copy_state_to_trial(mcba_ctx* ctx) {
  CK(cudaMemcpyAsync(ctx->trial.p, ctx->params.p, sizeof(double) * ctx->layout.len, cudaMemcpyDeviceToDevice, ctx->stream));
  return MCBA_OK;
}

LmArgs make_lm_args(mcba_ctx* ctx, int log_cap) {
  const DeviceProblem& P = ctx->P;
  LmArgs a{};
  a.P = P;
  a.trial = ctx->trial.p; a.state_len = (int)ctx->layout.len;
  a.n = P.n; a.n_s = P.n_s; a.F = P.F; a.fb = P.fb;
  a.n_items = P.C + P.B + P.F * P.npf + P.C + P.B * P.P + 2;
  a.Hss = ctx->Hss.p; a.Hff = ctx->Hff.p; a.W = ctx->W.p; a.g = ctx->g.p;
  a.frame_cost = ctx->frame_cost.p; a.lin_cost = ctx->lin_cost.p;
  a.x = ctx->x.p; a.x_new = ctx->x_new.p; a.sinv = ctx->sinv.p; a.d = ctx->d.p; a.gh = ctx->gh.p; a.gn = ctx->gn.p;
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

int launch_lm(mcba_ctx* ctx, const LmArgs& a) {
  const size_t sm = sizeof(double) * lm_smem_doubles(ctx->P.n_s, ctx->P.fb);
  LmArgs args = a;
#ifdef MCBA_SIMT_BUILD
  if (ctx->P.fb == 12) k_lm<12><<<ctx->lm_grid, LM_THREADS, sm, ctx->stream>>>(args); else k_lm<6><<<ctx->lm_grid, LM_THREADS, sm, ctx->stream>>>(args);
  CKL();
#else
  // cooperative launch: every CTA of the grid is resident for the whole kernel (the grid barriers spin)
  void* params[] = {&args};
  const void* fn = ctx->P.fb == 12 ? (const void*)k_lm<12> : (const void*)k_lm<6>;
  CK(cudaLaunchCooperativeKernel(fn, dim3(ctx->lm_grid), dim3(LM_THREADS), params, sm, ctx->stream));
  ctx->launches++;
#endif
  return MCBA_OK;
}

// one pass of the loop body: linearise the trial state, then accept / solve / step (k_lm)
int lm_body(mcba_ctx* ctx, int loss, double f_scale, const LmArgs& a) {
  int r = linearize(ctx, loss, f_scale, true); if (r) return r;
  return launch_lm(ctx, a);
}

int run_lm_loop(mcba_ctx* ctx, int loss, double f_scale, int log_cap) {
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
      int r = lm_body(ctx, loss, f_scale, a);
      ctx->stream = s;
      cudaError_t e = cudaStreamEndCapture(cap, nullptr);
      if (r) return r;
      if (e != cudaSuccess) { ctx->err = std::string("graph capture of the loop body: ") + cudaGetErrorString(e); return MCBA_ERR_CUDA; }
      CK(cudaGraphInstantiate(&ctx->sg.exec, g, 0));
      ctx->sg.key = key; ctx->sg.stream = s;
      ctx->sg.body_launches = ctx->launches - before;
    }
    ctx->launches = before;
    CK(cudaGraphLaunch(ctx->sg.exec, s));
    ctx->graph_launched = true;
    return MCBA_OK;
  }
#endif
  // host-driven loop (the SIMT interpreter build; MCBA_GRAPH=0): same kernels, one state read per body
  ctx->graph_launched = false;
  SolverState h{};
  for (int it = 0; it < log_cap + 8; it++) {
    int r = lm_body(ctx, loss, f_scale, a); if (r) return r;
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
  return MCBA_OK;
}

// the current and trial parameter state of `desc` (kept when they already fit: a re-selected table keeps its state); board_pts, if not
// null, receives where the uploads write the board points
int alloc_state(mcba_ctx* ctx, const mcba_problem_desc* desc, double** board_pts) {
  ctx->layout = state_layout(*desc);
  CK(ctx->params.alloc(ctx->layout.len)); CK(ctx->trial.alloc(ctx->layout.len));
  if (board_pts) *board_pts = ctx->params.p + ctx->layout.pts;
  return MCBA_OK;
}

// dimensions, variable layout, permutation and every solver buffer that depends on (C,F,B,P,N,V)
int setup_problem(mcba_ctx* ctx, const mcba_problem_desc* desc, int64_t N, int V, bool keep_state = false) {
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
  { int r = alloc_state(ctx, desc, nullptr); if (r) return r; }
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
    REQUIRE(lin_smem_for(P, warps) <= 220 * 1024, MCBA_ERR_UNSUPPORTED, "too many boards for the linearisation kernel's shared memory");
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
  CK(ctx->x.alloc(nn)); CK(ctx->x_new.alloc(nn)); CK(ctx->sinv.alloc(nn)); CK(ctx->d.alloc(nn)); CK(ctx->gh.alloc(nn)); CK(ctx->gn.alloc(nn));
  CK(ctx->S.alloc((size_t)std::max(P.n_s, 1) * std::max(P.n_s, 1))); CK(ctx->rhs.alloc((size_t)std::max(P.n_s, 1)));
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
  return MCBA_OK;
}
// MCBA_PROF=1: host wall clock at checkpoints of the upload path, on stderr (no synchronisation is added: it times what the host waits for)
struct UploadClock {
  bool on; std::chrono::steady_clock::time_point t0;
  explicit UploadClock(bool enabled) : on(enabled), t0(std::chrono::steady_clock::now()) {}
  void mark(const char* what) { if (on) fprintf(stderr, "[upload] %-28s %8.3f ms\n", what, std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count()); }
};
int check_desc(mcba_ctx* ctx, const mcba_problem_desc* desc) {
  REQUIRE(desc->C > 0 && desc->F >= 0 && desc->B > 0 && desc->P > 0, MCBA_ERR_ARG, "bad problem dimensions");
  REQUIRE(desc->P <= 65535, MCBA_ERR_UNSUPPORTED, "more than 65535 points per board");
  REQUIRE(desc->model >= 0 && desc->model <= 4, MCBA_ERR_ARG, "unknown camera model");
  REQUIRE(!((desc->optimize & MCBA_MOTION_ROLLING) && (desc->optimize & MCBA_MOTION_HAND_EYE)), MCBA_ERR_ARG, "more than one motion model");
  REQUIRE((int64_t)desc->C * desc->F * desc->B * desc->P < ((int64_t)1 << 31), MCBA_ERR_UNSUPPORTED, "more than 2^31 table entries per rank");
  return MCBA_OK;
}

// pack the resident dense table (ctx->dense_pts) under a device mask into the frame-major corner arrays the kernels read
// points_ready: event after which dense_pts holds the observations (they may still be in flight on the copy stream while the views are
// counted and scanned), or null
int pack_dense(mcba_ctx* ctx, const mcba_problem_desc* desc, const uint8_t* d_mask, bool keep_state, int64_t* n_corners,
               const uint8_t* d_view_valid = nullptr, cudaEvent_t points_ready = nullptr, bool points_f32 = false) {
  const int C = desc->C, F = desc->F, B = desc->B, Pn = desc->P;
  const int nv = C * F * B;
  cudaStream_t s = ctx->stream;
  CK(ctx->scan.alloc((size_t)3 * (nv + 1)));
  int* cnt_can = ctx->scan.p; int* cnt_fm = cnt_can + (nv + 1); int* flag_fm = cnt_fm + (nv + 1);
  int totals[2] = {0, 0};
  UploadClock clk(ctx->profiling);
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
  { int r = setup_problem(ctx, desc, N, V, keep_state); if (r) return r; }
  clk.mark("pack: setup_problem done");
  CK(cudaStreamSynchronize(s));
  clk.mark("pack: final synchronise");
  if (n_corners) *n_corners = N;
  ctx->uploaded = true;
  return MCBA_OK;
}

}  // namespace

// =====================================================================================================
extern "C" {

int mcba_version(void) { return 100; }

const char* mcba_last_error(const mcba_ctx* ctx) { return ctx ? ctx->err.c_str() : g_create_error.c_str(); }

int mcba_create(int device, mcba_ctx** out) {
  if (!out) return MCBA_ERR_ARG;
  *out = nullptr;
  int count = 0;
  cudaError_t e = cudaGetDeviceCount(&count);
  if (e != cudaSuccess || count == 0) { g_create_error = std::string("no CUDA device: ") + cudaGetErrorString(e); return MCBA_ERR_CUDA; }
  if (device < 0 || device >= count) { g_create_error = "device ordinal out of range"; return MCBA_ERR_ARG; }
  e = cudaSetDevice(device);
  if (e != cudaSuccess) { g_create_error = cudaGetErrorString(e); return MCBA_ERR_CUDA; }
  cudaDeviceProp prop;
  e = cudaGetDeviceProperties(&prop, device);
  if (e != cudaSuccess) { g_create_error = cudaGetErrorString(e); return MCBA_ERR_CUDA; }
  if (prop.major != 9 || prop.minor != 0) { g_create_error = "libmcba is built for sm_90a only (found sm_" + std::to_string(prop.major * 10 + prop.minor) + ")"; return MCBA_ERR_CUDA; }
  mcba_ctx* ctx = new mcba_ctx();
  ctx->device = device;
  ctx->num_sms = prop.multiProcessorCount;
  if (cudaStreamCreateWithFlags(&ctx->own_stream, cudaStreamNonBlocking) != cudaSuccess) { g_create_error = "cudaStreamCreate failed"; delete ctx; return MCBA_ERR_CUDA; }
  ctx->stream = ctx->own_stream;
  { const char* e = getenv("MCBA_GRAPH"); if (e && std::string(e) == "0") ctx->use_graph = false; }
  { const char* e = getenv("MCBA_PROF"); if (e && std::string(e) == "1") { ctx->profiling = true; ctx->use_graph = false; } }
  for (int model = MODEL_STANDARD; model <= MODEL_TILTED; model++)
    for (bool roll : {false, true})
      with_model(model, roll, [](auto M, auto R) {
        cudaFuncSetAttribute(k_linearize<decltype(M)::value, decltype(R)::value>, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024);
      });
  cudaFuncSetAttribute(k_reduce_shared<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
  cudaFuncSetAttribute(k_reduce_shared<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
  cudaFuncSetAttribute(k_lm<6>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
  cudaFuncSetAttribute(k_lm<12>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
  *out = ctx;
  return MCBA_OK;
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
  cudaStream_t own = ctx->own_stream;
  delete ctx;                            // device buffers are freed by their destructors
  if (own) cudaStreamDestroy(own);
}

int mcba_set_stream(mcba_ctx* ctx, void* stream) {
  if (!ctx) return MCBA_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  CK(cudaStreamSynchronize(ctx->stream));          // nothing of ours may still be in flight on the stream we leave
  ctx->stream = (cudaStream_t)stream;              // NULL is the legacy default stream (what torch reports as stream 0)
  return MCBA_OK;
}

int mcba_comm_unique_id(mcba_ctx* ctx, char out_id[128]) {
  // kept for the shape of the API (rank 0 makes an id, the host broadcasts it): the exchanges of a solve run inside the solver kernel over
  // NVLink peer mappings (mcba_peer_export / mcba_peer_import), there is no library communicator to create
  if (!ctx || !out_id) return MCBA_ERR_ARG;
  memset(out_id, 0, 128);
  snprintf(out_id, 128, "mcba-peer-group");
  return MCBA_OK;
}

int mcba_comm_init(mcba_ctx* ctx, const char id_[128], int rank, int world) {
  if (!ctx || !id_) return MCBA_ERR_ARG;
  REQUIRE(world >= 1 && world <= PEER_MAX_WORLD && rank >= 0 && rank < world, MCBA_ERR_ARG, "bad rank/world (1..16 ranks)");
  ctx->rank = rank; ctx->world = world; ctx->peer_ready = false;
  return MCBA_OK;
}

int mcba_peer_export(mcba_ctx* ctx, int64_t cap_doubles, char out_handle[64]) {
  if (!ctx || !out_handle) return MCBA_ERR_ARG;
  REQUIRE(ctx->world > 1 && ctx->world <= PEER_MAX_WORLD, MCBA_ERR_STATE, "peer buffers need an initialised communicator with 2..16 ranks");
  REQUIRE(cap_doubles > 0 && cap_doubles < ((int64_t)1 << 30), MCBA_ERR_ARG, "bad peer slot capacity");
  REQUIRE(sizeof(cudaIpcMemHandle_t) == 64, MCBA_ERR_UNSUPPORTED, "unexpected cudaIpcMemHandle_t size");
  CK(cudaSetDevice(ctx->device));
  if (ctx->peer_own) { cudaFree(ctx->peer_own); ctx->peer_own = nullptr; }
  ctx->peer_ready = false; ctx->peer_cap = (int)cap_doubles;
  const size_t bytes = peer_buffer_doubles(ctx->world, ctx->peer_cap) * sizeof(double);
  CK(cudaMalloc(&ctx->peer_own, bytes));
  CK(cudaMemset(ctx->peer_own, 0, bytes));
  CK(cudaDeviceSynchronize());
  cudaIpcMemHandle_t h;
  CK(cudaIpcGetMemHandle(&h, ctx->peer_own));
  memcpy(out_handle, &h, 64);
  return MCBA_OK;
}

int mcba_peer_import(mcba_ctx* ctx, const char* handles /* world x 64 bytes, rank order */) {
  if (!ctx || !handles) return MCBA_ERR_ARG;
  REQUIRE(ctx->peer_own != nullptr, MCBA_ERR_STATE, "mcba_peer_export has not been called");
  CK(cudaSetDevice(ctx->device));
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
  return MCBA_OK;
}

int mcba_upload(mcba_ctx* ctx, const mcba_problem_desc* desc, const int32_t* cam, const int32_t* frame,
                const int32_t* board, const int32_t* point, const double* obs, const double* board_points) {
  if (!ctx || !desc) return MCBA_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  const int C = desc->C, F = desc->F, B = desc->B, Pn = desc->P;
  const int64_t N = desc->N;
  { int r = check_desc(ctx, desc); if (r) return r; }
  REQUIRE(N >= 0 && N < ((int64_t)1 << 31), MCBA_ERR_UNSUPPORTED, "corner count out of range");
  REQUIRE(N == 0 || (cam && frame && board && point && obs), MCBA_ERR_ARG, "null corner arrays");
  REQUIRE(board_points != nullptr, MCBA_ERR_ARG, "null board points");
  ctx->table = false; ctx->table_selected = -1; ctx->errors_current = false;

  // ---- pack: stable counting sort of the canonical (c,f,b,p)-ordered corners by frame => (f,c,b,p) order
  std::vector<int64_t> fcount((size_t)F + 1, 0);
  for (int64_t k = 0; k < N; k++) {
    const int c = cam[k], f = frame[k], b = board[k], p = point[k];
    if (c < 0 || c >= C || f < 0 || f >= F || b < 0 || b >= B || p < 0 || p >= Pn) { ctx->err = "corner index out of range"; return MCBA_ERR_ARG; }
    fcount[(size_t)f + 1]++;
  }
  for (int f = 0; f < F; f++) fcount[(size_t)f + 1] += fcount[f];
  std::vector<uint32_t> order((size_t)N);
  {
    std::vector<int64_t> cursor(fcount.begin(), fcount.end() - 1);
    for (int64_t k = 0; k < N; k++) order[(size_t)cursor[frame[k]]++] = (uint32_t)k;
  }
  std::vector<double2> h_obs((size_t)N);
  std::vector<uint16_t> h_pid((size_t)N);
  std::vector<int> vstart, vcam, vframe, vboard, fvs((size_t)F + 1, 0);
  int prev_c = -1, prev_f = -1, prev_b = -1;
  for (int64_t i = 0; i < N; i++) {
    const uint32_t k = order[(size_t)i];
    h_obs[(size_t)i] = make_double2(obs[2 * (size_t)k], obs[2 * (size_t)k + 1]);
    h_pid[(size_t)i] = (uint16_t)point[k];
    const int c = cam[k], f = frame[k], b = board[k];
    if (c != prev_c || f != prev_f || b != prev_b) {
      vstart.push_back((int)i); vcam.push_back(c); vframe.push_back(f); vboard.push_back(b);
      prev_c = c; prev_f = f; prev_b = b;
    }
  }
  const int V = (int)vcam.size();
  vstart.push_back((int)N);
  {
    std::vector<int> cnt((size_t)F + 1, 0);
    for (int v = 0; v < V; v++) cnt[(size_t)vframe[v] + 1]++;
    for (int f = 0; f < F; f++) cnt[(size_t)f + 1] += cnt[f];
    fvs = cnt;
  }

#define UP(buf, vec) do { CK(ctx->buf.alloc((vec).size())); if (!(vec).empty()) CK(cudaMemcpyAsync(ctx->buf.p, (vec).data(), (vec).size() * sizeof((vec)[0]), cudaMemcpyHostToDevice, ctx->stream)); } while (0)
  UP(obs, h_obs); UP(pid, h_pid); UP(orig, order);
  UP(view_start, vstart); UP(view_cam, vcam); UP(view_frame, vframe); UP(view_board, vboard);
  UP(frame_view_start, fvs);
#undef UP
  double* bpts = nullptr;
  { int r = alloc_state(ctx, desc, &bpts); if (r) return r; }
  CK(cudaMemcpyAsync(bpts, board_points, sizeof(double) * (size_t)B * Pn * 3, cudaMemcpyHostToDevice, ctx->stream));
  { int r = setup_problem(ctx, desc, N, V); if (r) return r; }
  CK(cudaStreamSynchronize(ctx->stream));    // host staging vectors go out of scope
  ctx->uploaded = true;
  return MCBA_OK;
}

// Dense variant: the [C,F,B,P] inlier mask and [C,F,B,P,2] observations go to the device as they are and the
// packing (frame-major order, view records, canonical index map) happens there (pack_kernels.cuh).
namespace {
int upload_dense_any(mcba_ctx* ctx, const mcba_problem_desc* desc, const uint8_t* valid, const uint8_t* view_valid, const void* points, bool points_f32,
                     const double* board_points, int64_t* n_corners) {
  if (!ctx || !desc) return MCBA_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  { int r = check_desc(ctx, desc); if (r) return r; }
  REQUIRE(valid && points && board_points, MCBA_ERR_ARG, "null dense table");
  const int C = desc->C, F = desc->F, B = desc->B, Pn = desc->P;
  const int nv = C * F * B;
  const size_t dense = (size_t)nv * Pn;
  cudaStream_t s = ctx->stream;
  CK(ctx->dense_mask.alloc(std::max<size_t>(dense, 1)));
  if (points_f32) CK(ctx->dense_pts32.alloc(std::max<size_t>(dense, 1))); else CK(ctx->dense_pts.alloc(std::max<size_t>(dense, 1)));
  CK(ctx->view_valid.alloc(std::max<size_t>((size_t)nv, 1)));
  CK(ctx->scan.alloc((size_t)3 * (nv + 1)));
  double* bpts = nullptr;
  { int r = alloc_state(ctx, desc, &bpts); if (r) return r; }
  cudaEvent_t ready = nullptr;
  UploadClock clk(ctx->profiling);
  if (dense) {
    // the mask (1 B/point) goes first on the solver's stream; the observations (16 B/point) follow on the copy stream while the views
    // are counted and scanned, and the scatter waits for them
    CK(cudaMemcpyAsync(ctx->dense_mask.p, valid, dense, cudaMemcpyHostToDevice, s));
    if (view_valid) CK(cudaMemcpyAsync(ctx->view_valid.p, view_valid, (size_t)nv, cudaMemcpyHostToDevice, s));
    // the small copies from pageable memory go BEFORE the table: such a copy returns when it is done, and behind 100 MB on the copy engine
    // it would hold the host back until the table has crossed the link -- with it the count / scan kernels that should run beside it
    CK(cudaMemcpyAsync(bpts, board_points, sizeof(double) * (size_t)B * Pn * 3, cudaMemcpyHostToDevice, s));
    if (!ctx->copy_stream) { CK(cudaStreamCreateWithFlags(&ctx->copy_stream, cudaStreamNonBlocking)); CK(cudaEventCreateWithFlags(&ctx->copy_done, cudaEventDisableTiming)); CK(cudaEventCreateWithFlags(&ctx->copy_go, cudaEventDisableTiming)); }
    CK(cudaEventRecord(ctx->copy_go, s));                          // work queued on `s` before this call may still read dense_pts
    CK(cudaStreamWaitEvent(ctx->copy_stream, ctx->copy_go, 0));
    if (points_f32) CK(cudaMemcpyAsync(ctx->dense_pts32.p, points, dense * sizeof(float2), cudaMemcpyHostToDevice, ctx->copy_stream));
    else CK(cudaMemcpyAsync(ctx->dense_pts.p, points, dense * sizeof(double2), cudaMemcpyHostToDevice, ctx->copy_stream));
    CK(cudaEventRecord(ctx->copy_done, ctx->copy_stream));
    ready = ctx->copy_done;
    clk.mark("upload: copies issued");
  } else {
    CK(cudaMemcpyAsync(bpts, board_points, sizeof(double) * (size_t)B * Pn * 3, cudaMemcpyHostToDevice, s));
  }
  ctx->table = false; ctx->table_selected = -1; ctx->errors_current = false;
  return pack_dense(ctx, desc, ctx->dense_mask.p, false, n_corners, view_valid ? ctx->view_valid.p : nullptr, ready, points_f32);
}
}  // namespace

int mcba_upload_dense_views(mcba_ctx* ctx, const mcba_problem_desc* desc, const uint8_t* valid, const uint8_t* view_valid, const double* points,
                            const double* board_points, int64_t* n_corners) {
  return upload_dense_any(ctx, desc, valid, view_valid, points, false, board_points, n_corners);
}

int mcba_upload_dense_views_f32(mcba_ctx* ctx, const mcba_problem_desc* desc, const uint8_t* valid, const uint8_t* view_valid, const float* points,
                                const double* board_points, int64_t* n_corners) {
  return upload_dense_any(ctx, desc, valid, view_valid, points, true, board_points, n_corners);
}

int mcba_upload_dense(mcba_ctx* ctx, const mcba_problem_desc* desc, const uint8_t* mask, const double* points,
                      const double* board_points, int64_t* n_corners) {
  return mcba_upload_dense_views(ctx, desc, mask, nullptr, points, board_points, n_corners);
}

// ---------------------------------------------------------------------------------------------------------------
// Resident point table (include/mcba.h "resident point table"): Calibration.adjust_outliers without host round trips.

namespace {

int table_begin(mcba_ctx* ctx, const mcba_problem_desc* desc, const double* board_points, size_t* dense_out) {
  CK(cudaSetDevice(ctx->device));
  { int r = check_desc(ctx, desc); if (r) return r; }
  REQUIRE(board_points != nullptr, MCBA_ERR_ARG, "null board points");
  const size_t dense = (size_t)desc->C * desc->F * desc->B * desc->P;
  CK(ctx->valid_mask.alloc(std::max<size_t>(dense, 1))); CK(ctx->inlier_mask.alloc(std::max<size_t>(dense, 1)));
  CK(ctx->dense_pts.alloc(std::max<size_t>(dense, 1)));
  double* bpts = nullptr;
  { int r = alloc_state(ctx, desc, &bpts); if (r) return r; }
  CK(cudaMemcpyAsync(bpts, board_points, sizeof(double) * (size_t)desc->B * desc->P * 3, cudaMemcpyHostToDevice, ctx->stream));
  ctx->table = false; ctx->table_selected = -1; ctx->errors_current = false;
  *dense_out = dense;
  return MCBA_OK;
}

// inliers = valid, pack `valid`, remember the description
int table_finish(mcba_ctx* ctx, const mcba_problem_desc* desc, size_t dense, int64_t* n_valid) {
  if (dense) CK(cudaMemcpyAsync(ctx->inlier_mask.p, ctx->valid_mask.p, dense, cudaMemcpyDeviceToDevice, ctx->stream));
  ctx->table_desc = *desc;
  int64_t n = 0;
  { int r = pack_dense(ctx, desc, ctx->valid_mask.p, false, &n); if (r) return r; }
  ctx->table = true; ctx->table_selected = MCBA_TABLE_VALID;
  ctx->n_valid = n; ctx->n_inliers = n;
  if (n_valid) *n_valid = n;
  return MCBA_OK;
}

size_t table_dense(const mcba_ctx* ctx) {
  const mcba_problem_desc& d = ctx->table_desc;
  return (size_t)d.C * d.F * d.B * d.P;
}

int sort_errors(mcba_ctx* ctx, const double* in, double* out, int64_t n) {
  size_t bytes = 0;
  CK(cub::DeviceRadixSort::SortKeys(nullptr, bytes, in, out, n, 0, 64, ctx->stream));
  CK(ctx->sort_tmp.alloc(bytes));
  bytes = ctx->sort_tmp.n;
  CK(cub::DeviceRadixSort::SortKeys(ctx->sort_tmp.p, bytes, in, out, n, 0, 64, ctx->stream));
  ctx->launches += 4;
  return MCBA_OK;
}

}  // namespace

int mcba_table_upload(mcba_ctx* ctx, const mcba_problem_desc* desc, const uint8_t* valid, const double* points,
                      const double* board_points, int64_t* n_valid) {
  if (!ctx || !desc) return MCBA_ERR_ARG;
  REQUIRE(valid && points, MCBA_ERR_ARG, "null dense table");
  size_t dense = 0;
  { int r = table_begin(ctx, desc, board_points, &dense); if (r) return r; }
  if (dense) {
    CK(cudaMemcpyAsync(ctx->valid_mask.p, valid, dense, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(ctx->dense_pts.p, points, dense * sizeof(double2), cudaMemcpyHostToDevice, ctx->stream));
  }
  return table_finish(ctx, desc, dense, n_valid);
}

int mcba_table_from_detections(mcba_ctx* ctx, const mcba_problem_desc* desc, const int64_t* det_start, const int32_t* det_ids,
                               const double* det_xy, const double* board_points, int64_t* n_valid) {
  if (!ctx || !desc) return MCBA_ERR_ARG;
  REQUIRE(det_start != nullptr, MCBA_ERR_ARG, "null detection offsets");
  size_t dense = 0;
  { int r = table_begin(ctx, desc, board_points, &dense); if (r) return r; }
  const int nv = desc->C * desc->F * desc->B;
  const int64_t total = det_start[nv];
  REQUIRE(det_start[0] == 0 && total >= 0 && total < ((int64_t)1 << 31), MCBA_ERR_ARG, "bad detection offsets");
  REQUIRE(total == 0 || (det_ids && det_xy), MCBA_ERR_ARG, "null detection arrays");
  cudaStream_t s = ctx->stream;
  DevBuf<int64_t> d_start; DevBuf<int32_t> d_ids; DevBuf<double2> d_xy; DevBuf<int> d_bad;
  CK(d_start.alloc((size_t)nv + 1)); CK(d_ids.alloc((size_t)std::max<int64_t>(total, 1))); CK(d_xy.alloc((size_t)std::max<int64_t>(total, 1))); CK(d_bad.alloc(1));
  CK(cudaMemcpyAsync(d_start.p, det_start, sizeof(int64_t) * ((size_t)nv + 1), cudaMemcpyHostToDevice, s));
  if (total) {
    CK(cudaMemcpyAsync(d_ids.p, det_ids, sizeof(int32_t) * (size_t)total, cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(d_xy.p, det_xy, sizeof(double2) * (size_t)total, cudaMemcpyHostToDevice, s));
  }
  CK(cudaMemsetAsync(d_bad.p, 0, sizeof(int), s));
  if (dense) {
    CK(cudaMemsetAsync(ctx->valid_mask.p, 0, dense, s));
    CK(cudaMemsetAsync(ctx->dense_pts.p, 0, dense * sizeof(double2), s));    // fill_sparse leaves zeros where nothing was detected
  }
  int bad = 0;
  k_table_check_offsets<<<(nv + 1 + 255) / 256, 256, 0, s>>>(d_start.p, nv, total, d_bad.p); CKL();
  CK(cudaMemcpyAsync(&bad, d_bad.p, sizeof(int), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  REQUIRE(!bad, MCBA_ERR_ARG, "detection offsets are not a monotone CSR over C*F*B lists");
  if (nv > 0 && total > 0) {
    k_table_fill<<<(unsigned)(((size_t)nv * 32 + 255) / 256), 256, 0, s>>>(d_start.p, d_ids.p, d_xy.p, nv, desc->P, ctx->valid_mask.p, ctx->dense_pts.p, d_bad.p); CKL();
    CK(cudaMemcpyAsync(&bad, d_bad.p, sizeof(int), cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    REQUIRE(!bad, MCBA_ERR_ARG, "detection id outside [0, P)");
  }
  return table_finish(ctx, desc, dense, n_valid);
}

namespace {

// The caller's detection lists: list w = (c*F+f)*B+b of the C*F*B views holds point ids det_ids[det_start[w]:det_start[w+1]] in [0, P) and
// their pixel corners det_xy (a CSR layout); the boards' id grids are at most 64 x 64.
int check_detections(mcba_ctx* ctx, const mcba_problem_desc* desc, const int64_t* det_start, const int32_t* det_ids, const double* det_xy,
                     const int32_t* board_grid) {
  const int nv = desc->C * desc->F * desc->B;
  const int64_t total = det_start[nv];
  REQUIRE(det_start[0] == 0 && total >= 0 && total < ((int64_t)1 << 31), MCBA_ERR_ARG, "bad detection offsets");
  REQUIRE(total == 0 || (det_ids && det_xy), MCBA_ERR_ARG, "null detection arrays");
  for (int w = 0; w < nv; w++) REQUIRE(det_start[w + 1] >= det_start[w], MCBA_ERR_ARG, "detection offsets are not a monotone CSR over C*F*B lists");
  for (int64_t i = 0; i < total; i++) REQUIRE(det_ids[i] >= 0 && det_ids[i] < desc->P, MCBA_ERR_ARG, "detection id outside [0, P)");
  for (int b = 0; b < desc->B; b++)
    REQUIRE(board_grid[5 * b] > 0 && board_grid[5 * b + 1] > 0 && board_grid[5 * b + 2] > 0 && board_grid[5 * b] <= 64 && board_grid[5 * b + 1] <= 64,
            MCBA_ERR_UNSUPPORTED, "id grids are limited to 64 x 64 (bit masks of the occupied rows / columns)");
  return MCBA_OK;
}

// detection lists in that layout, the id grids and the board points -> ctx->pnp, with room for the outputs of k_pnp_views
int stage_detections(mcba_ctx* ctx, const mcba_problem_desc* desc, const int64_t* det_start, const int32_t* det_ids, const double* det_xy,
                     const int32_t* board_grid, const double* board_points) {
  const int nv = desc->C * desc->F * desc->B, B = desc->B, Pn = desc->P;
  const int64_t total = det_start[nv];
  cudaStream_t s = ctx->stream;
  auto& pb = ctx->pnp;
  const size_t tot = (size_t)std::max<int64_t>(total, 1);
  CK(pb.start.alloc((size_t)nv + 1)); CK(pb.ids.alloc(tot)); CK(pb.xy.alloc(tot)); CK(pb.und.alloc(tot)); CK(pb.grid.alloc((size_t)B * 5));
  CK(pb.bp.alloc((size_t)B * Pn * 3)); CK(pb.pose.alloc((size_t)nv * 16)); CK(pb.err.alloc(nv)); CK(pb.n.alloc(nv)); CK(pb.ok.alloc(nv));
  CK(cudaMemcpyAsync(pb.start.p, det_start, sizeof(int64_t) * ((size_t)nv + 1), cudaMemcpyHostToDevice, s));
  if (total) {
    CK(cudaMemcpyAsync(pb.ids.p, det_ids, sizeof(int32_t) * (size_t)total, cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(pb.xy.p, det_xy, sizeof(double2) * (size_t)total, cudaMemcpyHostToDevice, s));
  }
  CK(cudaMemcpyAsync(pb.grid.p, board_grid, sizeof(int32_t) * (size_t)B * 5, cudaMemcpyHostToDevice, s));
  CK(cudaMemcpyAsync(pb.bp.p, board_points, sizeof(double) * (size_t)B * Pn * 3, cudaMemcpyHostToDevice, s));
  return MCBA_OK;
}

// k_pnp_views over the staged lists: one warp per list, poses under the intrinsics intr [C][kint] (device) of camera model `model`
int launch_pnp(mcba_ctx* ctx, const mcba_problem_desc* desc, int model, int kint, const double* intr) {
  auto& pb = ctx->pnp;
  PnpArgs a{};
  a.C = desc->C; a.F = desc->F; a.B = desc->B; a.P = desc->P; a.model = model; a.kint = kint; a.nv = desc->C * desc->F * desc->B;
  a.det_start = pb.start.p; a.det_ids = pb.ids.p; a.det_xy = pb.xy.p; a.board_pts = pb.bp.p; a.intr = intr; a.grid = pb.grid.p;
  a.und = pb.und.p; a.poses = pb.pose.p; a.err = pb.err.p; a.npts = pb.n.p; a.valid = pb.ok.p; a.max_iters = 50;
  const int blocks = (a.nv + PNP_WARPS - 1) / PNP_WARPS;
  with_model(model, false, [&](auto M, auto) {
    constexpr int MODEL = decltype(M)::value;
    k_pnp_views<MODEL><<<blocks, PNP_WARPS * 32, 0, ctx->stream>>>(a);
  });
  CKL();
  return MCBA_OK;
}

}  // namespace

// Batched board-pose initialisation (pnp_kernels.cuh): one warp per detection list.  Independent of the uploaded problem.
int mcba_pnp_views(mcba_ctx* ctx, const mcba_problem_desc* desc, const int64_t* det_start, const int32_t* det_ids, const double* det_xy,
                   const double* board_points, const double* intrinsics, const int32_t* board_grid,
                   double* poses, double* errors, int32_t* num_points, uint8_t* valid) {
  if (!ctx || !desc) return MCBA_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  { int r = check_desc(ctx, desc); if (r) return r; }
  REQUIRE(det_start && board_points && intrinsics && board_grid && poses && errors && num_points && valid, MCBA_ERR_ARG, "null argument");
  const int nv = desc->C * desc->F * desc->B;
  if (nv == 0) return MCBA_OK;
  { int r = check_detections(ctx, desc, det_start, det_ids, det_xy, board_grid); if (r) return r; }
  const int kint = 5 + model_nd(desc->model);
  cudaStream_t s = ctx->stream;
  auto& pb = ctx->pnp;
  { int r = stage_detections(ctx, desc, det_start, det_ids, det_xy, board_grid, board_points); if (r) return r; }
  CK(pb.in.alloc((size_t)desc->C * kint));
  CK(cudaMemcpyAsync(pb.in.p, intrinsics, sizeof(double) * (size_t)desc->C * kint, cudaMemcpyHostToDevice, s));
  { int r = launch_pnp(ctx, desc, desc->model, kint, pb.in.p); if (r) return r; }
  CK(cudaMemcpyAsync(poses, pb.pose.p, sizeof(double) * 16 * (size_t)nv, cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(errors, pb.err.p, sizeof(double) * (size_t)nv, cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(num_points, pb.n.p, sizeof(int32_t) * (size_t)nv, cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(valid, pb.ok.p, (size_t)nv, cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  return MCBA_OK;
}

// Initialisation of single-camera intrinsic calibration (intrinsics_kernels.cuh): one homography per used view, K0 per camera
// (initIntrinsicParams2D), the initial per-view poses from k_pnp_views under K0 and zero distortion.  Independent of the uploaded problem.
int mcba_intrinsic_init(mcba_ctx* ctx, const mcba_problem_desc* desc, const int64_t* det_start, const int32_t* det_ids, const double* det_xy,
                        const double* board_points, const int32_t* board_grid, const int32_t* image_sizes, const uint8_t* view_use,
                        double* intrinsics, double* poses, uint8_t* ok) {
  if (!ctx || !desc) return MCBA_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  { int r = check_desc(ctx, desc); if (r) return r; }
  REQUIRE(det_start && board_points && board_grid && image_sizes && view_use && intrinsics && poses && ok, MCBA_ERR_ARG, "null argument");
  REQUIRE(desc->model != MODEL_FISHEYE, MCBA_ERR_UNSUPPORTED, "the intrinsic initialisation is for the pinhole camera models");
  const int C = desc->C, F = desc->F, B = desc->B, Pn = desc->P, nv = C * F * B;
  const int kint = 5 + model_nd(desc->model);
  { int r = check_detections(ctx, desc, det_start, det_ids, det_xy, board_grid); if (r) return r; }
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
  { int r = stage_detections(ctx, desc, start.data(), ids.data(), xy.data(), board_grid, board_points); if (r) return r; }
  CK(ib.used.alloc((size_t)std::max(n_used, 1))); CK(ib.cam_start.alloc((size_t)C + 1)); CK(ib.size.alloc((size_t)C * 2));
  CK(ib.H.alloc((size_t)std::max(n_used, 1) * 9)); CK(ib.hok.alloc((size_t)std::max(n_used, 1))); CK(ib.k0.alloc((size_t)C * kint));
  if (n_used) CK(cudaMemcpyAsync(ib.used.p, used.data(), sizeof(int32_t) * used.size(), cudaMemcpyHostToDevice, s));
  CK(cudaMemcpyAsync(ib.cam_start.p, cam_start.data(), sizeof(int32_t) * cam_start.size(), cudaMemcpyHostToDevice, s));
  CK(cudaMemcpyAsync(ib.size.p, image_sizes, sizeof(int32_t) * (size_t)C * 2, cudaMemcpyHostToDevice, s));
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
  if (nv) {
    { int r = launch_pnp(ctx, desc, MODEL_STANDARD, kint, ib.k0.p); if (r) return r; }      // zero distortion: the pinhole K0
    CK(cudaMemcpyAsync(poses, pb.pose.p, sizeof(double) * 16 * (size_t)nv, cudaMemcpyDeviceToHost, s));
    CK(cudaMemcpyAsync(ok, pb.ok.p, (size_t)nv, cudaMemcpyDeviceToHost, s));
  }
  CK(cudaMemcpyAsync(intrinsics, ib.k0.p, sizeof(double) * (size_t)C * kint, cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  return MCBA_OK;
}

// Per-view sums of squared pixel errors and corner counts of the packed problem at the current parameters (intrinsics_kernels.cuh)
int mcba_view_errors(mcba_ctx* ctx, double* sumsq, int64_t* count) {
  if (!ctx || !sumsq || !count) return MCBA_ERR_ARG;
  REQUIRE(ctx->uploaded, MCBA_ERR_STATE, "mcba_upload has not been called");
  CK(cudaSetDevice(ctx->device));
  DeviceProblem P = with_state(ctx, false);
  const size_t nv = (size_t)P.C * P.F * P.B;
  if (nv == 0) return MCBA_OK;
  int r = prepare(ctx, P); if (r) return r;
  DevBuf<double> ds; DevBuf<int64_t> dn;
  CK(ds.alloc(nv)); CK(dn.alloc(nv));
  cudaStream_t s = ctx->stream;
  CK(cudaMemsetAsync(ds.p, 0, sizeof(double) * nv, s)); CK(cudaMemsetAsync(dn.p, 0, sizeof(int64_t) * nv, s));
  if (P.V > 0) {
    ViewKernelArgs a{}; a.loss = MCBA_LOSS_LINEAR; a.f_scale = 1.0; a.view_cost = ctx->view_cost.p;
    r = launch_views<MODE_COST>(ctx, P, a); if (r) return r;
    k_view_sumsq<<<(P.V + 255) / 256, 256, 0, s>>>(P, ctx->view_cost.p, ds.p, dn.p);
    CKL();
  }
  CK(cudaMemcpyAsync(sumsq, ds.p, sizeof(double) * nv, cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(count, dn.p, sizeof(int64_t) * nv, cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  return MCBA_OK;
}

int mcba_table_download(mcba_ctx* ctx, uint8_t* valid, double* points) {
  if (!ctx) return MCBA_ERR_ARG;
  REQUIRE(ctx->table, MCBA_ERR_STATE, "no resident table (mcba_table_upload / mcba_table_from_detections)");
  CK(cudaSetDevice(ctx->device));
  const size_t dense = table_dense(ctx);
  if (valid && dense) CK(cudaMemcpyAsync(valid, ctx->valid_mask.p, dense, cudaMemcpyDeviceToHost, ctx->stream));
  if (points && dense) CK(cudaMemcpyAsync(points, ctx->dense_pts.p, dense * sizeof(double2), cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  return MCBA_OK;
}

int mcba_table_set_inliers(mcba_ctx* ctx, const uint8_t* mask) {
  if (!ctx) return MCBA_ERR_ARG;
  REQUIRE(ctx->table, MCBA_ERR_STATE, "no resident table (mcba_table_upload / mcba_table_from_detections)");
  CK(cudaSetDevice(ctx->device));
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
  return MCBA_OK;
}

int mcba_table_get_inliers(mcba_ctx* ctx, uint8_t* mask) {
  if (!ctx || !mask) return MCBA_ERR_ARG;
  REQUIRE(ctx->table, MCBA_ERR_STATE, "no resident table (mcba_table_upload / mcba_table_from_detections)");
  CK(cudaSetDevice(ctx->device));
  const size_t dense = table_dense(ctx);
  if (dense) CK(cudaMemcpyAsync(mask, ctx->inlier_mask.p, dense, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  return MCBA_OK;
}

int mcba_table_select(mcba_ctx* ctx, int which, int64_t* n_corners) {
  if (!ctx) return MCBA_ERR_ARG;
  REQUIRE(ctx->table, MCBA_ERR_STATE, "no resident table (mcba_table_upload / mcba_table_from_detections)");
  REQUIRE(which == MCBA_TABLE_VALID || which == MCBA_TABLE_INLIERS, MCBA_ERR_ARG, "unknown table selection");
  CK(cudaSetDevice(ctx->device));
  int64_t n = ctx->P.N;
  if (ctx->table_selected != which) {
    ctx->errors_current = false;
    const uint8_t* m = which == MCBA_TABLE_VALID ? ctx->valid_mask.p : ctx->inlier_mask.p;
    int r = pack_dense(ctx, &ctx->table_desc, m, true, &n); if (r) return r;
    ctx->table_selected = which;
    if (which == MCBA_TABLE_INLIERS) ctx->n_inliers = n;
  }
  if (n_corners) *n_corners = n;
  return MCBA_OK;
}

int mcba_table_errors(mcba_ctx* ctx, mcba_table_stats* stats) {
  if (!ctx) return MCBA_ERR_ARG;
  REQUIRE(ctx->table, MCBA_ERR_STATE, "no resident table (mcba_table_upload / mcba_table_from_detections)");
  { int r = mcba_table_select(ctx, MCBA_TABLE_VALID, nullptr); if (r) return r; }
  const DeviceProblem P = with_state(ctx, false);
  cudaStream_t s = ctx->stream;
  const int64_t N = P.N;
  double sums[3] = {0.0, 0.0, 0.0};
  if (N > 0) {
    CK(ctx->err_valid.alloc((size_t)N)); CK(ctx->err_sorted.alloc((size_t)N));
    CK(ctx->err_inl.alloc((size_t)N)); CK(ctx->err_inl_sorted.alloc((size_t)N));
    CK(ctx->table_part.alloc((size_t)3 * P.V + 3));
    { int r = prepare(ctx, P); if (r) return r; }
    ViewKernelArgs a{}; a.err = ctx->err_valid.p;
    { int r = launch_views<MODE_ERROR>(ctx, P, a); if (r) return r; }
    const int blocks = std::max(1, std::min((P.V + TABLE_WARPS - 1) / TABLE_WARPS, ctx->num_sms * 8));
    k_table_stats<<<blocks, TABLE_WARPS * 32, 0, s>>>(P, ctx->err_valid.p, ctx->inlier_mask.p, ctx->err_inl.p, ctx->table_part.p); CKL();
    double* d_sums = ctx->table_part.p + (size_t)3 * P.V;
    k_sum_partials<<<1, 1024, 0, s>>>(ctx->table_part.p, P.V, 3, 3, d_sums); CKL();
    CK(cudaMemcpyAsync(sums, d_sums, sizeof(sums), cudaMemcpyDeviceToHost, s));
    { int r = sort_errors(ctx, ctx->err_valid.p, ctx->err_sorted.p, N); if (r) return r; }
    { int r = sort_errors(ctx, ctx->err_inl.p, ctx->err_inl_sorted.p, N); if (r) return r; }
    CK(cudaStreamSynchronize(s));
  }
  ctx->n_valid = N; ctx->n_inliers = (int64_t)llround(sums[2]);
  ctx->errors_current = true;
  if (stats) { stats->n_valid = N; stats->n_inliers = ctx->n_inliers; stats->sumsq_valid = sums[0]; stats->sumsq_inliers = sums[1]; }
  return MCBA_OK;
}

int mcba_table_error_ranks(mcba_ctx* ctx, int which, const int64_t* ranks, int32_t n, double* out) {
  if (!ctx || (n > 0 && (!ranks || !out))) return MCBA_ERR_ARG;
  REQUIRE(ctx->table && ctx->errors_current, MCBA_ERR_STATE, "mcba_table_errors has not run since the parameters or the selection changed");
  REQUIRE(which == MCBA_TABLE_VALID || which == MCBA_TABLE_INLIERS, MCBA_ERR_ARG, "unknown table selection");
  if (n <= 0) return MCBA_OK;
  CK(cudaSetDevice(ctx->device));
  const int64_t count = which == MCBA_TABLE_VALID ? ctx->n_valid : ctx->n_inliers;
  for (int i = 0; i < n; i++) REQUIRE(ranks[i] >= 0 && ranks[i] < count, MCBA_ERR_ARG, "error rank out of range");
  CK(ctx->table_ranks.alloc((size_t)n)); CK(ctx->table_out.alloc((size_t)n));
  CK(cudaMemcpyAsync(ctx->table_ranks.p, ranks, sizeof(int64_t) * n, cudaMemcpyHostToDevice, ctx->stream));
  k_gather_ranks<<<(n + 127) / 128, 128, 0, ctx->stream>>>(which == MCBA_TABLE_VALID ? ctx->err_sorted.p : ctx->err_inl_sorted.p,
                                                         ctx->table_ranks.p, n, ctx->table_out.p); CKL();
  CK(cudaMemcpyAsync(out, ctx->table_out.p, sizeof(double) * n, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  return MCBA_OK;
}

int mcba_table_count_below(mcba_ctx* ctx, int which, const double* thresholds, int32_t n, int64_t* counts) {
  if (!ctx || (n > 0 && (!thresholds || !counts))) return MCBA_ERR_ARG;
  REQUIRE(ctx->table && ctx->errors_current, MCBA_ERR_STATE, "mcba_table_errors has not run since the parameters or the selection changed");
  REQUIRE(which == MCBA_TABLE_VALID || which == MCBA_TABLE_INLIERS, MCBA_ERR_ARG, "unknown table selection");
  if (n <= 0) return MCBA_OK;
  CK(cudaSetDevice(ctx->device));
  const int64_t count = which == MCBA_TABLE_VALID ? ctx->n_valid : ctx->n_inliers;
  CK(ctx->table_out.alloc((size_t)n)); CK(ctx->table_ranks.alloc((size_t)n));
  CK(cudaMemcpyAsync(ctx->table_out.p, thresholds, sizeof(double) * n, cudaMemcpyHostToDevice, ctx->stream));
  k_count_below<<<(n + 127) / 128, 128, 0, ctx->stream>>>(which == MCBA_TABLE_VALID ? ctx->err_sorted.p : ctx->err_inl_sorted.p, count,
                                                        ctx->table_out.p, n, ctx->table_ranks.p); CKL();
  CK(cudaMemcpyAsync(counts, ctx->table_ranks.p, sizeof(int64_t) * n, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  return MCBA_OK;
}

int mcba_table_reject(mcba_ctx* ctx, double threshold, int64_t* n_valid, int64_t* n_keep) {
  if (!ctx) return MCBA_ERR_ARG;
  REQUIRE(ctx->table && ctx->errors_current && ctx->table_selected == MCBA_TABLE_VALID, MCBA_ERR_STATE,
          "mcba_table_errors has not run since the parameters or the selection changed");
  CK(cudaSetDevice(ctx->device));
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
  return MCBA_OK;
}

int mcba_set_params(mcba_ctx* ctx, const double* cam_rt, const double* board_rt, const double* frame_rt, const double* intrinsics) {
  if (!ctx) return MCBA_ERR_ARG;
  REQUIRE(ctx->uploaded, MCBA_ERR_STATE, "mcba_upload has not been called");
  REQUIRE(cam_rt && board_rt && intrinsics && (frame_rt || ctx->P.F == 0 || ctx->P.fb == 0), MCBA_ERR_ARG, "null parameter array");
  const DeviceProblem& P = ctx->P;
  CK(cudaSetDevice(ctx->device));
  ctx->errors_current = false;
  CK(cudaMemcpyAsync(P.cam_rt, cam_rt, sizeof(double) * P.C * 6, cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemcpyAsync(P.board_rt, board_rt, sizeof(double) * P.B * 6, cudaMemcpyHostToDevice, ctx->stream));
  if (P.F && P.fb) CK(cudaMemcpyAsync(P.frame_rt, frame_rt, sizeof(double) * P.F * P.fb, cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemcpyAsync(P.intr, intrinsics, sizeof(double) * P.C * P.kint, cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  return MCBA_OK;
}

// Same state as 4x4 pose matrices (PoseSet.poses): the rotation-vector conversions of transform/rtvec.py run on the device.
// mats: f64[C+B+F][4][4] in the order cameras, boards, frames.
int mcba_set_state_matrices(mcba_ctx* ctx, const double* mats, const double* intrinsics) {
  if (!ctx) return MCBA_ERR_ARG;
  REQUIRE(ctx->uploaded, MCBA_ERR_STATE, "mcba_upload has not been called");
  REQUIRE(mats && intrinsics, MCBA_ERR_ARG, "null parameter array");
  const DeviceProblem& P = ctx->P;
  CK(cudaSetDevice(ctx->device));
  const int np = P.C + P.B + P.F;
  ctx->errors_current = false;
  CK(ctx->pose_mats.alloc((size_t)np * 16));
  CK(cudaMemcpyAsync(ctx->pose_mats.p, mats, sizeof(double) * 16 * np, cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemcpyAsync(P.intr, intrinsics, sizeof(double) * P.C * P.kint, cudaMemcpyHostToDevice, ctx->stream));
  k_matrices_to_state<<<(np + 127) / 128, 128, 0, ctx->stream>>>(P.C, P.B, P.F, ctx->pose_mats.p, P.cam_rt, P.board_rt, P.frame_rt, P.fb); CKL();
  CK(cudaStreamSynchronize(ctx->stream));     // the host arrays are borrowed only for the call
  return MCBA_OK;
}

int mcba_get_state_matrices(mcba_ctx* ctx, double* mats, double* intrinsics) {
  if (!ctx) return MCBA_ERR_ARG;
  REQUIRE(ctx->uploaded, MCBA_ERR_STATE, "mcba_upload has not been called");
  const DeviceProblem& P = ctx->P;
  CK(cudaSetDevice(ctx->device));
  const int np = P.C + P.B + P.F;
  if (mats) {
    CK(ctx->pose_mats.alloc((size_t)np * 16));
    const PoseT* derived = nullptr;
    if (P.motion == MOTION_HAND_EYE) { int r = prepare(ctx, with_state(ctx, false)); if (r) return r; derived = P.frame_T; }
    k_state_to_matrices<<<(np + 127) / 128, 128, 0, ctx->stream>>>(P.C, P.B, P.F, P.cam_rt, P.board_rt, P.frame_rt, ctx->pose_mats.p, P.fb, derived); CKL();
    CK(cudaMemcpyAsync(mats, ctx->pose_mats.p, sizeof(double) * 16 * np, cudaMemcpyDeviceToHost, ctx->stream));
  }
  if (intrinsics) CK(cudaMemcpyAsync(intrinsics, P.intr, sizeof(double) * P.C * P.kint, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  return MCBA_OK;
}

// RollingFrames (motion/rolling_frames.py:66-150): the frames of mcba_set_state_matrices are the start poses; the end poses
// f64[F][4][4] and the image heights f64[C] that turn an observed row into the blend weight (rolling_times, 15-19) come here.
int mcba_set_rolling(mcba_ctx* ctx, const double* end_pose_matrices, const double* image_heights) {
  if (!ctx) return MCBA_ERR_ARG;
  REQUIRE(ctx->uploaded, MCBA_ERR_STATE, "mcba_upload has not been called");
  const DeviceProblem& P = ctx->P;
  REQUIRE(P.motion == MOTION_ROLLING, MCBA_ERR_STATE, "the problem was not uploaded with MCBA_MOTION_ROLLING");
  REQUIRE((end_pose_matrices || P.F == 0) && image_heights, MCBA_ERR_ARG, "null parameter array");
  for (int c = 0; c < P.C; c++) REQUIRE(image_heights[c] > 0, MCBA_ERR_ARG, "image heights must be positive");
  CK(cudaSetDevice(ctx->device));
  ctx->errors_current = false;
  CK(cudaMemcpyAsync(ctx->img_h.p, image_heights, sizeof(double) * P.C, cudaMemcpyHostToDevice, ctx->stream));
  if (P.F) {
    CK(ctx->pose_mats.alloc((size_t)P.F * 16));
    CK(cudaMemcpyAsync(ctx->pose_mats.p, end_pose_matrices, sizeof(double) * 16 * P.F, cudaMemcpyHostToDevice, ctx->stream));
    // "cameras = 0, boards = 0, frames = F" view of the same kernel, writing the second half of every frame block
    k_matrices_to_state<<<(P.F + 127) / 128, 128, 0, ctx->stream>>>(0, 0, P.F, ctx->pose_mats.p, nullptr, nullptr, P.frame_rt + 6, 12); CKL();
  }
  CK(cudaStreamSynchronize(ctx->stream));
  return MCBA_OK;
}

int mcba_get_rolling(mcba_ctx* ctx, double* end_pose_matrices) {
  if (!ctx || !end_pose_matrices) return MCBA_ERR_ARG;
  REQUIRE(ctx->uploaded, MCBA_ERR_STATE, "mcba_upload has not been called");
  const DeviceProblem& P = ctx->P;
  REQUIRE(P.motion == MOTION_ROLLING, MCBA_ERR_STATE, "the problem was not uploaded with MCBA_MOTION_ROLLING");
  CK(cudaSetDevice(ctx->device));
  if (P.F) {
    CK(ctx->pose_mats.alloc((size_t)P.F * 16));
    k_state_to_matrices<<<(P.F + 127) / 128, 128, 0, ctx->stream>>>(0, 0, P.F, nullptr, nullptr, P.frame_rt + 6, ctx->pose_mats.p, 12, nullptr); CKL();
    CK(cudaMemcpyAsync(end_pose_matrices, ctx->pose_mats.p, sizeof(double) * 16 * P.F, cudaMemcpyDeviceToHost, ctx->stream));
  }
  CK(cudaStreamSynchronize(ctx->stream));
  return MCBA_OK;
}

// HandEye (motion/hand_eye.py:14-90): frame pose f = gripper_wrt_camera base_wrt_gripper[f] world_wrt_base; the arm poses are
// constants, the two outer transforms are the 12 motion parameters.  The frames of mcba_set_state_matrices are ignored.
int mcba_set_hand_eye(mcba_ctx* ctx, const double* base_wrt_gripper, const double* world_wrt_base, const double* gripper_wrt_camera) {
  if (!ctx) return MCBA_ERR_ARG;
  REQUIRE(ctx->uploaded, MCBA_ERR_STATE, "mcba_upload has not been called");
  const DeviceProblem& P = ctx->P;
  REQUIRE(P.motion == MOTION_HAND_EYE, MCBA_ERR_STATE, "the problem was not uploaded with MCBA_MOTION_HAND_EYE");
  REQUIRE((base_wrt_gripper || P.F == 0) && world_wrt_base && gripper_wrt_camera, MCBA_ERR_ARG, "null parameter array");
  CK(cudaSetDevice(ctx->device));
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
  return MCBA_OK;
}

int mcba_get_hand_eye(mcba_ctx* ctx, double* world_wrt_base, double* gripper_wrt_camera) {
  if (!ctx) return MCBA_ERR_ARG;
  REQUIRE(ctx->uploaded, MCBA_ERR_STATE, "mcba_upload has not been called");
  const DeviceProblem& P = ctx->P;
  REQUIRE(P.motion == MOTION_HAND_EYE, MCBA_ERR_STATE, "the problem was not uploaded with MCBA_MOTION_HAND_EYE");
  CK(cudaSetDevice(ctx->device));
  CK(ctx->pose_mats.alloc(32));
  k_state_to_matrices<<<1, 128, 0, ctx->stream>>>(0, 0, 2, nullptr, nullptr, P.he_rt, ctx->pose_mats.p, 6, nullptr); CKL();
  if (world_wrt_base) CK(cudaMemcpyAsync(world_wrt_base, ctx->pose_mats.p, sizeof(double) * 16, cudaMemcpyDeviceToHost, ctx->stream));
  if (gripper_wrt_camera) CK(cudaMemcpyAsync(gripper_wrt_camera, ctx->pose_mats.p + 16, sizeof(double) * 16, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  return MCBA_OK;
}

int mcba_get_params(mcba_ctx* ctx, double* cam_rt, double* board_rt, double* frame_rt, double* intrinsics) {
  if (!ctx) return MCBA_ERR_ARG;
  REQUIRE(ctx->uploaded, MCBA_ERR_STATE, "mcba_upload has not been called");
  const DeviceProblem& P = ctx->P;
  CK(cudaSetDevice(ctx->device));
  if (cam_rt) CK(cudaMemcpyAsync(cam_rt, P.cam_rt, sizeof(double) * P.C * 6, cudaMemcpyDeviceToHost, ctx->stream));
  if (board_rt) CK(cudaMemcpyAsync(board_rt, P.board_rt, sizeof(double) * P.B * 6, cudaMemcpyDeviceToHost, ctx->stream));
  if (frame_rt && P.F && P.fb) CK(cudaMemcpyAsync(frame_rt, P.frame_rt, sizeof(double) * P.F * P.fb, cudaMemcpyDeviceToHost, ctx->stream));
  if (intrinsics) CK(cudaMemcpyAsync(intrinsics, P.intr, sizeof(double) * P.C * P.kint, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  return MCBA_OK;
}

int mcba_num_params(mcba_ctx* ctx, int64_t* n) {
  if (!ctx || !n) return MCBA_ERR_ARG;
  REQUIRE(ctx->uploaded, MCBA_ERR_STATE, "mcba_upload has not been called");
  *n = ctx->P.n;
  return MCBA_OK;
}

static int read_x_canonical(mcba_ctx* ctx, double* x) {
  const DeviceProblem& P = ctx->P;
  if (P.n == 0) return MCBA_OK;
  k_gather_params<<<(P.n + 255) / 256, 256, 0, ctx->stream>>>(P, ctx->x.p, P.cam_rt, P.board_rt, P.frame_rt, P.intr); CKL();
  std::vector<double> h((size_t)P.n);
  CK(cudaMemcpyAsync(h.data(), ctx->x.p, sizeof(double) * P.n, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  for (int i = 0; i < P.n; i++) x[ctx->perm[(size_t)i]] = h[(size_t)i];
  return MCBA_OK;
}
static int write_x_canonical(mcba_ctx* ctx, const double* x, double* dev_x) {
  const DeviceProblem& P = ctx->P;
  if (P.n == 0) return MCBA_OK;
  std::vector<double> h((size_t)P.n);
  for (int i = 0; i < P.n; i++) h[(size_t)i] = x[ctx->perm[(size_t)i]];
  CK(cudaMemcpyAsync(dev_x, h.data(), sizeof(double) * P.n, cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  return MCBA_OK;
}

int mcba_get_param_vec(mcba_ctx* ctx, double* x) {
  if (!ctx || !x) return MCBA_ERR_ARG;
  REQUIRE(ctx->uploaded, MCBA_ERR_STATE, "mcba_upload has not been called");
  CK(cudaSetDevice(ctx->device));
  return read_x_canonical(ctx, x);
}

int mcba_set_param_vec(mcba_ctx* ctx, const double* x) {
  if (!ctx || !x) return MCBA_ERR_ARG;
  REQUIRE(ctx->uploaded, MCBA_ERR_STATE, "mcba_upload has not been called");
  CK(cudaSetDevice(ctx->device));
  ctx->errors_current = false;
  int r = write_x_canonical(ctx, x, ctx->x.p); if (r) return r;
  r = set_state_from_x(ctx, ctx->x.p, false); if (r) return r;
  CK(cudaStreamSynchronize(ctx->stream));
  return MCBA_OK;
}

int mcba_residuals(mcba_ctx* ctx, const double* x, double* r_out, double* cost) {
  if (!ctx) return MCBA_ERR_ARG;
  REQUIRE(ctx->uploaded, MCBA_ERR_STATE, "mcba_upload has not been called");
  CK(cudaSetDevice(ctx->device));
  bool trial = false;
  if (x) {
    // evaluate at x without disturbing the stored parameters: trial state = current state overwritten by x
    int r = copy_state_to_trial(ctx); if (r) return r;
    r = write_x_canonical(ctx, x, ctx->x_new.p); if (r) return r;
    r = set_state_from_x(ctx, ctx->x_new.p, true); if (r) return r;
    trial = true;
  } else {
    int r = prepare(ctx, with_state(ctx, false)); if (r) return r;
  }
  DeviceProblem P = with_state(ctx, trial);
  if (r_out && P.N > 0) {
    DevBuf<double> dr; CK(dr.alloc((size_t)2 * P.N));
    ViewKernelArgs a{}; a.resid = dr.p;
    int r = launch_views<MODE_RESID>(ctx, P, a); if (r) return r;
    CK(cudaMemcpyAsync(r_out, dr.p, sizeof(double) * 2 * P.N, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
  }
  if (cost) {
    int r = trial_cost(ctx, 0, 1.0, trial); if (r) return r;
    CK(cudaMemcpyAsync(cost, ctx->eval_cost.p, sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
  }
  return MCBA_OK;
}

int mcba_reprojection_error(mcba_ctx* ctx, double* err) {
  if (!ctx || !err) return MCBA_ERR_ARG;
  REQUIRE(ctx->uploaded, MCBA_ERR_STATE, "mcba_upload has not been called");
  CK(cudaSetDevice(ctx->device));
  DeviceProblem P = with_state(ctx, false);
  if (P.N == 0) return MCBA_OK;
  int r = prepare(ctx, P); if (r) return r;
  DevBuf<double> de; CK(de.alloc((size_t)P.N));
  ViewKernelArgs a{}; a.err = de.p;
  r = launch_views<MODE_ERROR>(ctx, P, a); if (r) return r;
  CK(cudaMemcpyAsync(err, de.p, sizeof(double) * P.N, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  return MCBA_OK;
}

int mcba_linearize(mcba_ctx* ctx, const double* x, double* JtJ, double* Jtr, double* cost) {
  if (!ctx) return MCBA_ERR_ARG;
  REQUIRE(ctx->uploaded, MCBA_ERR_STATE, "mcba_upload has not been called");
  CK(cudaSetDevice(ctx->device));
  const DeviceProblem& P = ctx->P;
  if (x) { int r = mcba_set_param_vec(ctx, x); if (r) return r; }
  else { int r = prepare(ctx, with_state(ctx, false)); if (r) return r; }
  int r = linearize(ctx, 0, 1.0); if (r) return r;
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
  return MCBA_OK;
}

int mcba_solve(mcba_ctx* ctx, const mcba_solve_opts* opts, mcba_solve_result* result, mcba_log_row* log, int32_t log_capacity) {
  if (!ctx || !opts || !result) return MCBA_ERR_ARG;
  REQUIRE(ctx->uploaded, MCBA_ERR_STATE, "mcba_upload has not been called");
  REQUIRE(opts->loss >= 0 && opts->loss <= 4, MCBA_ERR_ARG, "unknown loss");
  REQUIRE(opts->max_nfev > 0, MCBA_ERR_ARG, "max_nfev must be positive");
  REQUIRE(opts->f_scale > 0, MCBA_ERR_ARG, "f_scale must be positive");
  REQUIRE(ctx->world == 1 || ctx->peer_ready, MCBA_ERR_STATE, "several ranks: the exchanges run over NVLink peer memory (mcba_peer_export / mcba_peer_import first)");
  CK(cudaSetDevice(ctx->device));
  const DeviceProblem& P = ctx->P;
  REQUIRE(ctx->world == 1 || (size_t)P.n_s * P.n_s + 2 * (size_t)P.n_s + 16 <= (size_t)ctx->peer_cap, MCBA_ERR_STATE,
          "the reduced normal equations do not fit the NVLink exchange slots: export larger peer buffers (mcba_peer_export cap >= n_s^2 + 2 n_s + 16)");
  cudaStream_t s = ctx->stream;
  const int n = P.n;
  memset(result, 0, sizeof(*result));
  ctx->launches = 0;
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
  int r;
  if (n == 0) {      // nothing to optimise: report the cost and leave
    r = prepare(ctx, with_state(ctx, false)); if (r) return r;
    r = linearize(ctx, opts->loss, opts->f_scale); if (r) return r;
    if (ctx->world > 1) {       // one number: the host's collective is the simplest exchange (no solver state involved)
      ctx->err = "nothing to optimise on several ranks: sum mcba_residuals' cost on the host"; return MCBA_ERR_UNSUPPORTED;
    }
    CK(cudaMemcpyAsync(&h.cost, ctx->lin_cost.p, sizeof(double), cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    result->initial_cost = h.cost; result->cost = h.cost; result->nfev = 1; result->njev = 1; result->status = 1;
    if (log && log_capacity > 0) { log[0] = mcba_log_row{0, 1, h.cost, NAN, NAN, 0.0}; result->n_log = 1; }
    CK(cudaEventRecord(ev.b, s)); CK(cudaEventSynchronize(ev.b));
    float ms0 = 0; cudaEventElapsedTime(&ms0, ev.a, ev.b);
    result->device_ms = ms0; result->kernel_launches = ctx->launches;
    return MCBA_OK;
  }
  CK(cudaMemcpyAsync(ctx->state.p, &h, sizeof(h), cudaMemcpyHostToDevice, s));
  // x0 and the trial state := the current state; its pose tables
  k_gather_params<<<(n + 255) / 256, 256, 0, s>>>(P, ctx->x.p, P.cam_rt, P.board_rt, P.frame_rt, P.intr); CKL();
  CK(cudaMemcpyAsync(ctx->x_new.p, ctx->x.p, sizeof(double) * n, cudaMemcpyDeviceToDevice, s));
  r = copy_state_to_trial(ctx); if (r) return r;
  r = prepare(ctx, with_state(ctx, true)); if (r) return r;
  const int cap = std::max(8, opts->max_nfev + 4);
  CK(ctx->dev_log.alloc((size_t)cap));

  r = run_lm_loop(ctx, opts->loss, opts->f_scale, cap); if (r) return r;

  CK(cudaMemcpyAsync(&h, ctx->state.p, sizeof(h), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  if (h.status == -2) { ctx->err = "Residuals are not finite in the initial point."; return MCBA_ERR_NONFINITE; }
  if (h.status == -3) { ctx->err = "a peer rank did not answer an in-kernel exchange (timeout): the ranks left mcba_solve out of step"; return MCBA_ERR_NCCL; }
  const int nlog = std::min(h.nlog, cap);
  std::vector<mcba_log_row> rows((size_t)std::max(nlog, 1));
  if (nlog > 0) CK(cudaMemcpyAsync(rows.data(), ctx->dev_log.p, sizeof(mcba_log_row) * nlog, cudaMemcpyDeviceToHost, s));
  // leave the context consistent: pose tables of the final (current) state
  r = prepare(ctx, with_state(ctx, false)); if (r) return r;
  CK(cudaEventRecord(ev.b, s));
  CK(cudaEventSynchronize(ev.b));
  float ms = 0; cudaEventElapsedTime(&ms, ev.a, ev.b);
  if (nlog > 0) result->initial_cost = rows[0].cost;
  if (log) for (int i = 0; i < nlog && i < log_capacity; i++) log[i] = rows[(size_t)i];
  result->cost = h.cost; result->optimality = h.g_norm; result->nfev = h.nfev; result->njev = h.njev;
  result->status = h.status == -99 ? 0 : h.status; result->n_log = std::min(nlog, (int)log_capacity); result->device_ms = ms;
  if (ctx->graph_launched) ctx->launches += ctx->sg.body_launches * h.nfev;      // the WHILE node ran the body once per evaluation
  result->kernel_launches = ctx->launches; result->chol_retries = h.chol_fail;
  return MCBA_OK;
}

int mcba_bench_info(mcba_ctx* ctx, int which, int64_t* corners, int64_t* bytes, int32_t* launches) {
  if (!ctx) return MCBA_ERR_ARG;
  REQUIRE(ctx->uploaded, MCBA_ERR_STATE, "mcba_upload has not been called");
  const DeviceProblem& P = ctx->P;
  int64_t per_corner = 18, per_view = 16, l = 1;
  if (which == MCBA_BENCH_RESIDUAL) per_corner = 18 + 4 + 16;
  if (corners) *corners = P.N;
  if (bytes) *bytes = per_corner * P.N + per_view * P.V;      // per launch
  if (launches) *launches = (int32_t)l;
  return MCBA_OK;
}

int mcba_bench_launch(mcba_ctx* ctx, int which, int repeats) {
  if (!ctx) return MCBA_ERR_ARG;
  REQUIRE(ctx->uploaded, MCBA_ERR_STATE, "mcba_upload has not been called");
  CK(cudaSetDevice(ctx->device));
  DeviceProblem P = with_state(ctx, false);
  int r;
  if (!(which & MCBA_BENCH_NO_PREPARE)) { r = prepare(ctx, P); if (r) return r; }
  which &= ~MCBA_BENCH_NO_PREPARE;
  for (int i = 0; i < repeats; i++) {
    ViewKernelArgs a{}; a.loss = 0; a.f_scale = 1.0;
    if (which == MCBA_BENCH_LINEARIZE) r = launch_linearize(ctx, P, 0, 1.0);
    else if (which == MCBA_BENCH_COST) { a.view_cost = ctx->view_cost.p; r = launch_views<MODE_COST>(ctx, P, a); }
    else { ctx->err = "unsupported bench kernel"; return MCBA_ERR_ARG; }
    if (r) return r;
  }
  return MCBA_OK;
}

}  // extern "C"
