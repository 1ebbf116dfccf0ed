// solver_kernels.cuh — on-device trust-region machinery: the solver state and the scalar steps of
// scipy.optimize._lsq.trf.trf_no_bounds (the solver behind calibration.py:209-210): jac scaling bookkeeping
// (common.py compute_jac_scale), damping from the 1-D Cauchy model, the 2-D subspace trust-region step,
// ratio test / radius update (update_tr_radius), termination tests (check_termination).  The phases that use
// them -- and the Schur-complement solve -- are the persistent kernel of lm_kernel.cuh.
// The one deliberate change: scipy's LSMR inner iteration is replaced by an EXACT solve of
//     (A + reg I) gn = g_h ,   A = D H D  (H = J^T J block-arrow: shared | per-frame 6x6)
// through the Schur complement of the per-frame blocks (S = A_ss + reg I - sum_f Y_f Y_f^T).
#pragma once
#include "kernels.cuh"

namespace mcba {

struct SolverState {
  double ftol, xtol, gtol, reg_floor;
  int max_nfev;
  int nfev, njev, iteration, status, accepted, first_scale, chol_fail, done;
  double cost, cost_new, Delta, reg;
  double g_norm, gh_norm;
  double alpha, beta;            // step_h = alpha*gh + beta*gn
  double B11, B12, B22, gS1, gS2, n1, n2, mu;
  double step_h_norm, predicted, step_norm, x_norm, actual_reduction, ratio;
  double last_step_norm, last_reduction;
  // device-resident loop (lm_kernel.cuh)
  int pending, step_parts, nlog, pad_;       // a trial state waits for its acceptance test | per-CTA step records | rows logged
  double step2_s, xn2_s, agg;                // shared (replicated) parts of ||step||^2 and ||x||^2 of the pending trial; g_h^T A g_h
};

// ---- NVLink peer-memory exchange of k_lm (lm_kernel.cuh LmPeer): layout of the per-rank buffers
constexpr int PEER_MAX_WORLD = 16;
constexpr int PEER_FLAG_STRIDE = 8;      // doubles (64 B) between flags

__host__ __device__ inline size_t peer_flag_off(int world, int parity, int src) { return (size_t)(parity * world + src) * PEER_FLAG_STRIDE; }
__host__ __device__ inline size_t peer_data_off(int world, int cap, int parity, int src) {
  return (size_t)2 * world * PEER_FLAG_STRIDE + ((size_t)parity * world + src) * cap;
}
__host__ __device__ inline size_t peer_buffer_doubles(int world, int cap) { return (size_t)2 * world * PEER_FLAG_STRIDE + (size_t)2 * world * cap; }

__device__ __forceinline__ double block_sum(double v, double* sm) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  __syncthreads();
  if (lane == 0) sm[w] = v;
  __syncthreads();
  double r = 0.0;
  if (w == 0) {
    r = lane < nw ? sm[lane] : 0.0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) r += __shfl_xor_sync(0xffffffffu, r, o);
  }
  return r;   // valid in thread 0
}

// ---- bulk asynchronous copies (the 1-D form of the Tensor Memory Accelerator, cp.async.bulk) with an mbarrier as completion signal:
// data travels HBM/L2 -> shared memory without passing through registers, several transfers in flight per CTA (k_linearize: the pose
// tables of the next frame; k_lm: the operand tiles of the Schur SYRK, a four-stage pipeline).
__device__ __forceinline__ unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long* bar, unsigned count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long* bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, unsigned bytes, unsigned long long* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, unsigned phase) {
  asm volatile("{ .reg .pred p_; MBW_: mbarrier.try_wait.parity.shared::cta.b64 p_, [%0], %1; @p_ bra.uni MBD_; bra.uni MBW_; MBD_: }"
               ::"r"(smem_u32(bar)), "r"(phase) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
// generic-proxy writes to shared memory (plain stores) before the async proxy (bulk copies) touches the same bytes
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// deterministic sum of per-CTA partials: out[j] = sum_i part[i*stride + j]
__global__ void k_sum_partials(const double* part, int count, int stride, int nout, double* out) {
  __shared__ double sm[32];
  for (int j = 0; j < nout; j++) {
    double s = 0.0;
    for (int i = threadIdx.x; i < count; i += blockDim.x) s += part[(size_t)i * stride + j];
    s = block_sum(s, sm);
    if (threadIdx.x == 0) out[j] = s;
    __syncthreads();
  }
}

// trf.py top of the outer loop: ||g||_inf, gtol / max_nfev exits, first-iteration cost and Delta.
// Every sum below is split into its shared (_s) and frame (_f) part; the frame parts are summed over the ranks.
__device__ inline void begin_iteration(SolverState* st, double gh2_s, double gh2_f, double gmax_s, double gmax_f, double xs2_s, double xs2_f,
                                       double cost) {
  const double gh2 = gh2_s + gh2_f;
  st->gh_norm = sqrt(gh2);
  st->g_norm = fmax(gmax_s, gmax_f);
  if (st->first_scale) {
    st->cost = cost;
    double D0 = sqrt(xs2_s + xs2_f);
    st->Delta = (D0 == 0.0) ? 1.0 : D0;
    st->first_scale = 0;
  }
  if (st->g_norm < st->gtol) st->status = 1;
  st->done = (st->status != -99) || (st->nfev >= st->max_nfev);
}

// trf.py: reg_term = -ag_value / Delta^2 with ag_value = min over [0, Delta/||g_h||] of a t^2 + b t,
// a = g_h^T A g_h, b = -||g_h||^2 (build_quadratic_1d / minimize_quadratic_1d).
__device__ inline void reg_compute(SolverState* st, double a) {
  const double gh2 = st->gh_norm * st->gh_norm;
  const double b = -gh2;
  const double ub = st->Delta / st->gh_norm;
  // minimize a t^2 + b t on [0, ub]
  double best = 0.0;
  { const double yv = a * ub * ub + b * ub; if (yv < best) best = yv; }
  if (a != 0.0) { const double ext = -0.5 * b / a; if (ext > 0.0 && ext < ub) { const double yv = a * ext * ext + b * ext; if (yv < best) best = yv; } }
  double reg = -best / (st->Delta * st->Delta);
  if (!(reg > st->reg_floor)) reg = st->reg_floor;
  st->reg = reg;
}


// shapes shared by the phases of lm_kernel.cuh
constexpr int SYRK_TILE = 32;
__host__ __device__ constexpr int syrk_fr(int fb) { return 48 / fb; }       // frames staged per step: 2 x 12 KB of shared memory
constexpr int CHOL_SMALL_MAX = 127;      // reduced systems up to this size are factored by one CTA with the matrix in registers (row n = right-hand side)
constexpr int CHOL_NB = 32;              // panel width of the cooperative blocked factorisation above it

// trf.py: S = qr([g_h, gn_h]); B_S = (J_h S)^T (J_h S); g_S = S^T g_h   -- expressed through Gram-Schmidt
// coefficients so that no basis vectors are materialised: q1 = gh/n1, q2 = (gn - mu q1)/n2.
__device__ inline void subspace_compute(SolverState* st, double agg, double agn, double ann, double dot_s, double dot_f, double gn2_s, double gn2_f) {
  const double n1 = st->gh_norm;
  const double dot = dot_s + dot_f;
  const double gn2 = gn2_s + gn2_f;
  const double mu = dot / n1;
  double n2sq = gn2 - mu * mu;
  st->n1 = n1; st->mu = mu;
  st->B11 = agg / (n1 * n1);
  st->gS1 = n1; st->gS2 = 0.0;
  if (!(n2sq > 1e-28 * gn2) || !(n2sq > 0.0)) {     // gn parallel to gh: 1-D subspace
    st->n2 = 0.0; st->B12 = 0.0; st->B22 = 1.0;
  } else {
    const double n2 = sqrt(n2sq), c = mu / n1;
    st->n2 = n2;
    st->B12 = (agn - c * agg) / (n1 * n2);
    st->B22 = (ann - 2.0 * c * agn + c * c * agg) / (n2 * n2);
  }
}


// common.py solve_trust_region_2d: minimise 0.5 p^T B p + g^T p, ||p|| <= Delta  (B 2x2 symmetric).
// Interior Newton point if B is positive definite and inside; otherwise the global boundary minimiser via
// the secular equation in the eigenbasis of B (equivalent to scipy's argmin over the quartic's real roots).
__host__ __device__ inline void solve_tr_2d(double b11, double b12, double b22, double g1, double g2, double Delta, double& p1, double& p2) {
  const double det = b11 * b22 - b12 * b12;
  if (b11 > 0.0 && det > 0.0) {
    const double q1 = -(b22 * g1 - b12 * g2) / det, q2 = -(b11 * g2 - b12 * g1) / det;
    if (q1 * q1 + q2 * q2 <= Delta * Delta) { p1 = q1; p2 = q2; return; }
  }
  // eigen-decomposition
  const double tr = b11 + b22, df = b11 - b22;
  const double rad = sqrt(df * df + 4.0 * b12 * b12);
  const double l1 = 0.5 * (tr - rad), l2 = 0.5 * (tr + rad);       // l1 <= l2
  double v1x, v1y;
  if (fabs(b12) > 1e-300 * fmax(fabs(tr), 1.0)) { v1x = l1 - b22; v1y = b12; const double nn = hypot(v1x, v1y); if (nn > 0) { v1x /= nn; v1y /= nn; } else { v1x = 1; v1y = 0; } }
  else if (b11 <= b22) { v1x = 1; v1y = 0; } else { v1x = 0; v1y = 1; }
  const double v2x = -v1y, v2y = v1x;
  const double h1 = v1x * g1 + v1y * g2, h2 = v2x * g1 + v2y * g2;
  // find sigma >= max(0,-l1) with h1^2/(l1+s)^2 + h2^2/(l2+s)^2 = Delta^2
  const double gnorm = hypot(h1, h2);
  double lo = fmax(0.0, -l1);
  double hi = fmax(lo, gnorm / Delta - l1) + 1e-300;
  auto pn2 = [&](double s) { const double a = h1 / (l1 + s), b = h2 / (l2 + s); return a * a + b * b; };
  double c1, c2;
  // hard case: h1 ~ 0 and the l2-component alone stays inside at s = -l1
  const bool hard = (fabs(h1) <= 1e-14 * gnorm) && (l2 + lo > 0.0) && (h2 * h2 / ((l2 + lo) * (l2 + lo)) <= Delta * Delta);
  if (hard || gnorm == 0.0) {
    c2 = (l2 + lo > 0.0) ? -h2 / (l2 + lo) : 0.0;
    const double rem = Delta * Delta - c2 * c2;
    c1 = sqrt(fmax(rem, 0.0));
  } else {
    while (pn2(hi) > Delta * Delta) hi = 2.0 * hi + 1e-12;
    double s = hi;
    for (int it = 0; it < 200; it++) {
      s = 0.5 * (lo + hi);
      if (pn2(s) > Delta * Delta) lo = s; else hi = s;
      if (hi - lo <= 1e-16 * fmax(hi, 1e-300)) break;
    }
    s = 0.5 * (lo + hi);
    c1 = -h1 / (l1 + s); c2 = -h2 / (l2 + s);
    const double nn = hypot(c1, c2);
    if (nn > 0.0) { c1 *= Delta / nn; c2 *= Delta / nn; }
  }
  p1 = c1 * v1x + c2 * v2x;
  p2 = c1 * v1y + c2 * v2y;
}

__device__ inline void tr_step_compute(SolverState* st) {
  double p1, p2;
  solve_tr_2d(st->B11, st->B12, st->B22, st->gS1, st->gS2, st->Delta, p1, p2);
  if (st->n2 == 0.0) p2 = 0.0;
  st->step_h_norm = sqrt(p1 * p1 + p2 * p2);
  st->predicted = -(0.5 * (st->B11 * p1 * p1 + 2.0 * st->B12 * p1 * p2 + st->B22 * p2 * p2) + st->gS1 * p1 + st->gS2 * p2);
  // step_h = p1 q1 + p2 q2 = alpha gh + beta gn
  if (st->n2 == 0.0) { st->alpha = p1 / st->n1; st->beta = 0.0; }
  else { st->beta = p2 / st->n2; st->alpha = p1 / st->n1 - st->beta * st->mu / st->n1; }
}

// trf.py inner loop after fun(x_new): actual reduction, update_tr_radius, check_termination (one thread)
__device__ inline void accept_compute(SolverState* st, double cost_new, double step2_s, double step2_f, double xn2_s, double xn2_f) {
  st->nfev += 1;
  st->cost_new = cost_new;
  const double shn = st->step_h_norm;
  if (!isfinite(cost_new)) {            // trf.py: non-finite f_new -> shrink and retry
    st->Delta = 0.25 * shn;
    st->actual_reduction = -1.0;
    st->accepted = 0;
    return;
  }
  const double actual = st->cost - cost_new;
  const double pred = st->predicted;
  double ratio;
  if (pred > 0.0) ratio = actual / pred; else if (pred == 0.0 && actual == 0.0) ratio = 1.0; else ratio = 0.0;
  double Dn = st->Delta;
  if (ratio < 0.25) Dn = 0.25 * shn;
  else if (ratio > 0.75 && shn > 0.95 * st->Delta) Dn = 2.0 * st->Delta;
  const double step_norm = sqrt(step2_s + step2_f);
  const double x_norm = sqrt(xn2_s + xn2_f);
  st->step_norm = step_norm; st->x_norm = x_norm; st->actual_reduction = actual; st->ratio = ratio;
  const bool ft = (actual < st->ftol * st->cost) && (ratio > 0.25);
  const bool xt = step_norm < st->xtol * (st->xtol + x_norm);
  int status = -99;
  if (ft && xt) status = 4; else if (ft) status = 2; else if (xt) status = 3;
  st->status = status;
  if (status == -99) st->Delta = Dn;
  st->accepted = actual > 0.0;
}

}  // namespace mcba
