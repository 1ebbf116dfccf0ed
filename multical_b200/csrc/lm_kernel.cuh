// lm_kernel.cuh — the trust-region iteration as ONE persistent cooperative kernel per trial step.
//
// Round 1 ran the solver phase of an LM iteration as ~12 launches (k_scale, k_quad, k_schur_frames, k_schur_syrk, k_chol_small,
// k_backsub, k_dots, k_quad, k_step, k_make_trial, k_accept ...) of 5-50 us each, every one a chain of a few dependent L2 round trips,
// plus one host synchronisation per trial.  k_lm does all of it in one launch: the grid (<= one CTA per SM, all co-resident) walks the
// phases below separated by grid barriers (an arrive counter and a generation word in L2, ~1 us), the scalar trust-region logic of
// scipy's trf_no_bounds runs REPLICATED in every CTA on a shared-memory copy of the state (identical inputs, identical arithmetic:
// no broadcast needed), and the accept / reject decision, the iteration log and the loop condition stay on the device.  The host
// enqueues  [k_linearize -> k_reduce_shared -> k_lm]  as the body of a CUDA-graph WHILE node and reads the result once per SOLVE.
//
//   phase A  accept / reject the pending trial (cost from the per-frame costs of the fused linearisation at the trial point)
//   phase B  Jacobian scaling (x_scale='jac'), g_h, ||g||_inf                        -> barrier -> begin-of-iteration (termination tests, log row)
//   phase C  g_h^T A g_h on the block structure                                     -> barrier -> damping `reg` (1-D Cauchy model)
//   phase D  per frame: L L^T = D H_ff D + reg I, Y_f, z_f ; S = D H_ss D           -> barrier
//   phase E  S -= sum_f Y_f Y_f^T, rhs -= sum_f Y_f z_f: tile x frame-chunk partials -> barrier -> fixed-order sum over the chunks -> barrier
//   phase F  reduced solve (S + reg I) gn_s = rhs + g_h,s                            -> barrier
//   phase G  per frame: back-substitution gn_f, then the quadratic forms / dots of the 2-D subspace {g_h, gn}    -> barrier -> 2x2 model
//   phase I  trust-region step in the subspace, x_new                                -> barrier -> trial parameter state + pose tables
// Several GPUs (frames sharded): the four exchanges of an iteration (trial cost + next gradient/diagonal | g_h^T A g_h | S, rhs |
// subspace sums) run INSIDE the kernel over NVLink peer memory (exchange() below), in rank order -> identical values on every rank.
#pragma once
#include "solver_kernels.cuh"

namespace mcba {

constexpr int LM_THREADS = 256;
constexpr int LM_WARPS = LM_THREADS / 32;

__device__ __forceinline__ unsigned long long lm_ld_volatile(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.volatile.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void lm_st_volatile(unsigned long long* p, unsigned long long v) {
  asm volatile("st.volatile.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}

// Grid barrier: bar[0] = arrive counter, bar[1] = generation.  All CTAs of the launch are co-resident (cooperative launch, grid <= SMs).
// `spins` bounds the wait (a rank that left the solve early must not hang its peers' GPUs): on overflow *err is set and the wait ends.
__device__ __forceinline__ void grid_barrier(unsigned long long* bar, unsigned nblocks) {
  __syncthreads();
  if (threadIdx.x == 0 && nblocks > 1) {
    __threadfence();
    const unsigned long long g = lm_ld_volatile(bar + 1);
    const unsigned long long t = atomicAdd(bar, 1ull);
    if (t == (unsigned long long)nblocks - 1) {
      atomicExch(bar, 0ull);
      __threadfence();
      lm_st_volatile(bar + 1, g + 1);
    } else {
      while (lm_ld_volatile(bar + 1) == g) { }
    }
    __threadfence();
  }
  __syncthreads();
}

// 1/sqrt(x) for x in [1e-30, 1e30]: single-precision seed + two Newton steps in double (relative error ~1e-7 -> ~2e-14 -> < 1e-16).
// A dozen instructions on the critical path of a Cholesky column instead of the ~40 of the library routine (measured: the pivot warp's
// INSTRUCTION COUNT, at ~5 cycles per dependent issue, is what a column costs -- not the fp64 latencies).
__device__ __forceinline__ double fast_rsqrt(double x) {
  double r = (double)rsqrtf((float)x);
  double e = fma(-x * r, r, 1.0);
  r = fma(0.5 * r, e, r);
  e = fma(-x * r, r, 1.0);
  return fma(0.5 * r, e, r);
}

struct LmPeer {                      // NVLink peer-memory exchange (one buffer per rank, IPC-mapped into every rank; layout of peer_allreduce.cuh)
  int rank, world, cap;
  double* base[PEER_MAX_WORLD];
  unsigned long long* seq;           // device counter of the exchanges done so far (same on every rank)
  long long timeout_cycles;          // bound on the wait for a peer's flag
};

struct LmArgs {
  DeviceProblem P;                   // parameter pointers = the CURRENT state; pose tables = the state last linearised (the trial)
  double* trial; int state_len;      // TRIAL parameter state (what k_linearize reads): the layout of the current one, state_len doubles
  int n, n_s, F, fb, n_items;
  // linearisation at the trial point (k_linearize + k_reduce_shared [+ add-on kernels])
  const double* Hss; const double* Hff; const double* W; const double* g; const double* frame_cost; const double* lin_cost;
  // iteration vectors
  double *x, *x_new, *sinv, *d, *gh, *gn;
  // Schur complement
  double *Y, *Lf, *zf, *S, *rhs, *Spart, *rpart, *Linv;
  int syrk_chunks, syrk_cf;
  // partial sums (indexed by frame / virtual block: independent of the grid size where it matters for reproducibility)
  double *part_scale, *part_quad, *part_step;
  SolverState* st;
  mcba_log_row* log; int log_cap;
  unsigned long long* bar;
  LmPeer peer;
  unsigned long long cond_handle; int use_cond;      // CUDA-graph WHILE node: the kernel sets the loop condition itself
  unsigned long long* prof;          // MCBA_PROF=1: %globaltimer at the phase boundaries of the last launch (CTA 0), else null
};

// ---------------------------------------------------------------- replicated block-wide sums
// deterministic: fixed thread -> element map, fixed tree.  Result valid in EVERY thread (broadcast through shared memory).
__device__ __forceinline__ double block_sum_all(double v, double* sm) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  __syncthreads();
  if (lane == 0) sm[w] = v;
  __syncthreads();
  double r = 0.0;
#pragma unroll
  for (int i = 0; i < LM_WARPS; i++) r += sm[i];
  return r;
}
__device__ __forceinline__ double block_max_all(double v, double* sm) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  __syncthreads();
  if (lane == 0) sm[w] = v;
  __syncthreads();
  double r = 0.0;
#pragma unroll
  for (int i = 0; i < LM_WARPS; i++) r = fmax(r, sm[i]);
  return r;
}
// sum of count records part[i*stride + j] over i, every CTA in the same order
__device__ __forceinline__ double sum_records(const double* part, int count, int stride, int j, double* sm) {
  double s = 0.0;
  for (int i = threadIdx.x; i < count; i += LM_THREADS) s += __ldcg(&part[(size_t)i * stride + j]);
  return block_sum_all(s, sm);
}
__device__ __forceinline__ double max_records(const double* part, int count, int stride, int j, double* sm) {
  double s = 0.0;
  for (int i = threadIdx.x; i < count; i += LM_THREADS) s = fmax(s, __ldcg(&part[(size_t)i * stride + j]));
  return block_max_all(s, sm);
}

// ---------------------------------------------------------------- in-kernel all-reduce over NVLink peer memory
// All CTAs of all ranks call it with the same segment list.  push (slice-parallel remote stores into my slot on every rank) -> grid
// barrier -> one thread publishes this rank's sequence flag on every rank -> every CTA waits for all ranks' flags -> reduce in rank
// order (slice-parallel) -> grid barrier.  Two parities of slots: a rank cannot start exchange k+2 before every rank finished k.
struct XSeg { double* buf; int count; int op; };      // op 0 = sum, 1 = max
__device__ inline void exchange(const LmArgs& a, const XSeg* seg, int nseg, unsigned long long seq, int* err) {
  const LmPeer& pr = a.peer;
  const int parity = (int)(seq & 1ull);
  int total = 0;
  for (int s = 0; s < nseg; s++) total += seg[s].count;
  const size_t slot = peer_data_off(pr.world, pr.cap, parity, pr.rank);
  for (int idx = blockIdx.x * LM_THREADS + threadIdx.x; idx < total; idx += gridDim.x * LM_THREADS) {
    int s = 0, off = idx;
    while (off >= seg[s].count) { off -= seg[s].count; s++; }
    const double v = __ldcg(seg[s].buf + off);
    for (int p = 0; p < pr.world; p++) pr.base[p][slot + idx] = v;
  }
  __threadfence_system();
  grid_barrier(a.bar, gridDim.x);
  if (blockIdx.x == 0 && threadIdx.x < pr.world) {
    __threadfence_system();
    lm_st_volatile(reinterpret_cast<unsigned long long*>(pr.base[threadIdx.x] + peer_flag_off(pr.world, parity, pr.rank)), seq);
  }
  if (threadIdx.x < pr.world) {
    const unsigned long long* f = reinterpret_cast<const unsigned long long*>(pr.base[pr.rank] + peer_flag_off(pr.world, parity, threadIdx.x));
    const long long t0 = clock64();
    while (lm_ld_volatile(f) != seq) {
      if (pr.timeout_cycles > 0 && clock64() - t0 > pr.timeout_cycles) { *err = 1; break; }
    }
  }
  __syncthreads();
  __threadfence_system();
  const double* mine = pr.base[pr.rank];
  for (int idx = blockIdx.x * LM_THREADS + threadIdx.x; idx < total; idx += gridDim.x * LM_THREADS) {
    int s = 0, off = idx;
    while (off >= seg[s].count) { off -= seg[s].count; s++; }
    double acc = __ldcv(mine + peer_data_off(pr.world, pr.cap, parity, 0) + idx);
    for (int src = 1; src < pr.world; src++) {
      const double v = __ldcv(mine + peer_data_off(pr.world, pr.cap, parity, src) + idx);
      acc = seg[s].op == 0 ? acc + v : fmax(acc, v);
    }
    seg[s].buf[off] = acc;
  }
  __threadfence();
  grid_barrier(a.bar, gridDim.x);
}

// ---------------------------------------------------------------- phase bodies
// per frame (one warp): L L^T = D_f H_ff D_f + reg I ; Y_f = (D_s W_f D_f) L^-T ; z_f = L^-1 gh_f
template <int FB>
__device__ __forceinline__ void schur_frame(const LmArgs& a, int f, double reg, int lane, double* Lw /*[FB*FB + FB] shared, per warp*/) {
  // the stored factor keeps 1 / L_ii on its diagonal: every substitution below (and the back-substitution of phase G) multiplies
  const int n_s = a.n_s;
  double* L = Lw; double* df = Lw + FB * FB;
  if (lane == 0) {
    const double* H = a.Hff + (size_t)f * FB * FB;
    double A[FB * FB];
#pragma unroll
    for (int j = 0; j < FB; j++) df[j] = a.d[n_s + FB * f + j];
#pragma unroll
    for (int i = 0; i < FB; i++)
#pragma unroll
      for (int j = 0; j < FB; j++) A[i * FB + j] = df[i] * df[j] * H[i * FB + j] + (i == j ? reg : 0.0);
    double Lr[FB * FB];
#pragma unroll
    for (int j = 0; j < FB; j++) {
      double s = A[j * FB + j];
#pragma unroll
      for (int k = 0; k < FB; k++) if (k < j) s -= Lr[j * FB + k] * Lr[j * FB + k];
      const double rs = fast_rsqrt(fmin(fmax(s, 1e-30), 1e30));
      Lr[j * FB + j] = rs;                                  // 1 / L_jj
#pragma unroll
      for (int i = 0; i < FB; i++) {
        if (i > j) {
          double t = A[i * FB + j];
#pragma unroll
          for (int k = 0; k < FB; k++) if (k < j) t -= Lr[i * FB + k] * Lr[j * FB + k];
          Lr[i * FB + j] = t * rs;
        } else if (i < j) Lr[i * FB + j] = 0.0;
      }
    }
    double z[FB];
#pragma unroll
    for (int i = 0; i < FB; i++) {
      double t = a.gh[n_s + FB * f + i];
#pragma unroll
      for (int k = 0; k < FB; k++) if (k < i) t -= Lr[i * FB + k] * z[k];
      z[i] = t * Lr[i * FB + i];
      a.zf[(size_t)f * FB + i] = z[i];
    }
#pragma unroll
    for (int i = 0; i < FB * FB; i++) { L[i] = Lr[i]; a.Lf[(size_t)f * FB * FB + i] = Lr[i]; }
  }
  __syncwarp();
  const double* Wf = a.W + (size_t)f * n_s * FB;
  double* Yf = a.Y + (size_t)f * SYRK_TILE * FB;        // tile-major: row s of frame f at y_offset(F, FB, f, s)
  const size_t ytile = (size_t)a.F * SYRK_TILE * FB;
#pragma unroll 2
  for (int s = lane; s < n_s; s += 32) {
    const double ds = a.d[s];
    double y[FB], wr[FB];
    {
      const double2* w2 = reinterpret_cast<const double2*>(Wf + (size_t)s * FB);
#pragma unroll
      for (int i = 0; i < FB / 2; i++) { const double2 w = w2[i]; wr[2 * i] = w.x; wr[2 * i + 1] = w.y; }
    }
#pragma unroll
    for (int i = 0; i < FB; i++) {
      double t = ds * wr[i] * df[i];
#pragma unroll
      for (int k = 0; k < FB; k++) if (k < i) t -= L[i * FB + k] * y[k];
      y[i] = t * L[i * FB + i];
    }
    double2* y2 = reinterpret_cast<double2*>(Yf + (size_t)(s >> 5) * ytile + (size_t)(s & 31) * FB);
#pragma unroll
    for (int i = 0; i < FB / 2; i++) y2[i] = make_double2(y[2 * i], y[2 * i + 1]);
  }
  __syncwarp();
}

// one 32x32 tile (ti <= tj) of sum_f Y_f Y_f^T over a frame chunk -> Spart[chunk], diagonal tiles also sum_f Y_f z_f -> rpart[chunk].
// Operands: Y is tile-major ([row tile][frame][32][FB], rows beyond n_s zero), so the frames of a step (48 k-columns: 8 frames x 6, or
// 4 x 12) are ONE contiguous piece per operand: a step is two bulk asynchronous copies (cp.async.bulk + mbarrier) of 12 KB straight into
// shared memory, SYRK_STAGES steps in flight per CTA.  (Frame-major Y needed a copy per frame and operand, 16 per step, and a step then
// cost what the copy unit takes to work off 16 requests, whatever their size; before that, register-prefetched operands: one HBM/L2
// round trip per step.)
// Product on the fp64 tensor path, bound by the fragment loads from shared memory, not by the DMMAs: warp w owns the 16 x 16 block
// (w & 3) of the tile and every second k-step (w >> 2) -- 4 fragment loads feed 4 DMMAs (8 x 16 blocks over all k-steps: 3 loads per 2)
// -- and the rows a lane group reads are permuted (group g -> row 2 (g & 3) + (g >> 2)) so that with 6 doubles per row the 16 lanes of a
// half-warp hit 16 different 8-byte banks (rows 0..3 of a plain fragment collide two ways).  The two k-halves are added in a fixed order.
constexpr int SYRK_K = 48;
constexpr int SYRK_STAGES = 4;
template <int FB> __host__ __device__ constexpr int syrk_stage_doubles() { return 2 * SYRK_K * SYRK_TILE; }      // Yi | Yj, each [SYRK_FR][32][FB]
template <int FB>
__device__ __forceinline__ void syrk_tile(const LmArgs& a, int ti, int tj, int chunk, double* sh /* SYRK_STAGES * 2 * 48 * 32 doubles */, unsigned long long* sbar, unsigned& phases) {
  constexpr int SYRK_FR = syrk_fr(FB);
  static_assert(SYRK_FR * FB == SYRK_K && SYRK_FR <= LM_WARPS, "a step stages 48 k-columns; one warp per frame slot for the rhs");
  constexpr int FR_DOUBLES = SYRK_TILE * FB;                 // one frame's rows of a tile
  constexpr int STAGE = 2 * SYRK_K * SYRK_TILE;
  const int n_s = a.n_s, F = a.F;
  const int f0 = chunk * a.syrk_cf, f1 = min(F, f0 + a.syrk_cf);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, grp = lane >> 2, tig = lane & 3;
  const int qd = warp & 3, I2 = qd >> 1, J2 = qd & 1, kh = warp >> 2;
  const int pg = 2 * (grp & 3) + (grp >> 2);                 // row of the 8-row fragment this lane group reads
  const int nsteps = (f1 - f0 + SYRK_FR - 1) / SYRK_FR;
  double c[8];
#pragma unroll
  for (int q = 0; q < 8; q++) c[q] = 0.0;
  double racc = 0.0;
  __syncthreads();                                            // every warp has left the previous tile's stages
  fence_proxy_async();                                        // (also orders the previous phase's plain stores to this buffer before the copies)
  __syncthreads();
  auto issue = [&](int step) {                                // thread 0: the copies of one step into stage step % SYRK_STAGES
    const int st = step % SYRK_STAGES;
    const int fbase = f0 + step * SYRK_FR, nf = min(SYRK_FR, f1 - fbase);
    double* Yi = sh + (size_t)st * STAGE; double* Yj = Yi + SYRK_K * SYRK_TILE;
    const unsigned bytes = (unsigned)(nf * FR_DOUBLES * sizeof(double));
    mbar_expect_tx(&sbar[st], 2 * bytes);
    bulk_g2s(Yi, a.Y + ((size_t)ti * F + fbase) * FR_DOUBLES, bytes, &sbar[st]);
    bulk_g2s(Yj, a.Y + ((size_t)tj * F + fbase) * FR_DOUBLES, bytes, &sbar[st]);
  };
  if (tid == 0) for (int s0 = 0; s0 < SYRK_STAGES - 1 && s0 < nsteps; s0++) issue(s0);
  for (int step = 0; step < nsteps; step++) {
    const int st = step % SYRK_STAGES;
    if (tid == 0 && step + SYRK_STAGES - 1 < nsteps) issue(step + SYRK_STAGES - 1);      // its stage was consumed in step - 1 (barrier below)
    mbar_wait(&sbar[st], (phases >> st) & 1u);
    phases ^= 1u << st;
    const double* Yi = sh + (size_t)st * STAGE; const double* Yj = Yi + SYRK_K * SYRK_TILE;
    const int fbase = f0 + step * SYRK_FR, nf = min(SYRK_FR, f1 - fbase);
#pragma unroll
    for (int ks2 = 0; ks2 < SYRK_K / 8; ks2++) {
      const int ks = 2 * ks2 + kh;
      const int kidx = 4 * ks + tig, ff = kidx / FB, k = kidx % FB;          // k-column -> (frame of the step, component)
      const double* yi = Yi + ff * FR_DOUBLES + (16 * I2 + pg) * FB + k;
      const double* yj = Yj + ff * FR_DOUBLES + (16 * J2 + pg) * FB + k;
      // a chunk's last step may hold fewer frames than a stage: what lies behind them is a previous step's data, not zeros
      const bool on = ff < nf;
      const double fa0 = on ? yi[0] : 0.0, fa1 = on ? yi[8 * FB] : 0.0, fb0 = on ? yj[0] : 0.0, fb1 = on ? yj[8 * FB] : 0.0;
      dmma884(c[0], c[1], fa0, fb0);
      dmma884(c[2], c[3], fa0, fb1);
      dmma884(c[4], c[5], fa1, fb0);
      dmma884(c[6], c[7], fa1, fb1);
    }
    if (ti == tj) {                                           // rhs: thread (row = tid % 32, frame slot = tid / 32 (+ 8 for 4-frame steps: none))
      const int r = tid & 31, ff = tid >> 5;
      if (ff < nf) {
        const double* z = a.zf + (size_t)(fbase + ff) * FB;
#pragma unroll
        for (int k = 0; k < FB; k++) racc += Yi[ff * FR_DOUBLES + r * FB + k] * z[k];
      }
    }
    __syncthreads();                                          // the stage may be refilled
  }
  double* Sp = a.Spart + (size_t)chunk * n_s * n_s;
  if (ti == tj) {                                             // the frame slots' partial sums, added in slot order
    sh[tid] = racc;
    __syncthreads();
    if (tid < SYRK_TILE) {
      double r8 = 0.0;
#pragma unroll
      for (int q = 0; q < LM_WARPS; q++) r8 += sh[q * 32 + tid];
      const int i = ti * SYRK_TILE + tid;
      if (i < n_s) a.rpart[(size_t)chunk * n_s + i] = r8;
    }
    __syncthreads();
  }
  // the second k-half's fragments go through shared memory to the warp that owns the same block and are added there
  if (kh == 1) {
#pragma unroll
    for (int q = 0; q < 8; q++) sh[(qd * 8 + q) * 32 + lane] = c[q];
  }
  __syncthreads();
  if (kh == 0) {
#pragma unroll
    for (int q = 0; q < 8; q++) c[q] += sh[(qd * 8 + q) * 32 + lane];
    const int p0 = 2 * ((2 * tig) & 3) + ((2 * tig) >> 2), p1 = 2 * ((2 * tig + 1) & 3) + ((2 * tig + 1) >> 2);      // columns of the C fragment's two entries
#pragma unroll
    for (int ra = 0; ra < 2; ra++)
#pragma unroll
      for (int cb = 0; cb < 2; cb++) {
        const int i = ti * SYRK_TILE + 16 * I2 + 8 * ra + pg;
        const int jb = tj * SYRK_TILE + 16 * J2 + 8 * cb;
        if (i < n_s) {
          if (jb + p0 < n_s) Sp[(size_t)i * n_s + jb + p0] = c[(2 * ra + cb) * 2];
          if (jb + p1 < n_s) Sp[(size_t)i * n_s + jb + p1] = c[(2 * ra + cb) * 2 + 1];
        }
      }
  }
}

// ---- blocked right-looking Cholesky for n_s > CHOL_SMALL_MAX, NB = 32 panels, the grid cooperating between barriers.
// The diagonal block by ONE warp: lane i keeps row i in registers, a column is one shuffle of the pivot, one rsqrt and a
// shuffle per trailing column -- no block barrier on the column path (scripts/chol_bench.cu times it against the
// 256-thread version, whose column costs two __syncthreads).  The inverse of the factor follows in the same warp, lane j solving
// for column j with four independent partial sums per row.
__device__ __noinline__ void chol_diag_warp_body(int n, int kb, double* S, double* Linv_all, int* chol_fail, double* sh) {
  double (*Lm)[CHOL_NB + 1] = reinterpret_cast<double (*)[CHOL_NB + 1]>(sh);
  double (*Liv)[CHOL_NB + 1] = reinterpret_cast<double (*)[CHOL_NB + 1]>(sh + CHOL_NB * (CHOL_NB + 1));
  const int nb = min(CHOL_NB, n - kb);
  const int tid = threadIdx.x;
  __syncthreads();                       // the block may just have been updated by this CTA (look-ahead tile of the previous panel)
  {
    // all of a thread's loads first, then the stores: through the generic pointers of this function the compiler has to keep a load behind
    // the shared-memory store that precedes it, and the four L2 round trips would queue up one behind the other
    double v[CHOL_NB * CHOL_NB / LM_THREADS];
#pragma unroll
    for (int q = 0; q < CHOL_NB * CHOL_NB / LM_THREADS; q++) {
      const int o = tid + LM_THREADS * q, i = o / CHOL_NB, j = o % CHOL_NB;
      v[q] = (i < nb && j < nb) ? (j <= i ? __ldcg(&S[(size_t)(kb + i) * n + kb + j]) : 0.0) : (i == j ? 1.0 : 0.0);
    }
#pragma unroll
    for (int q = 0; q < CHOL_NB * CHOL_NB / LM_THREADS; q++) { const int o = tid + LM_THREADS * q; Lm[o / CHOL_NB][o % CHOL_NB] = v[q]; }
  }
  __syncthreads();
  if (tid < 32) {
    const int lane = tid;
    double a[CHOL_NB], rsd[CHOL_NB];
#pragma unroll
    for (int j = 0; j < CHOL_NB; j++) a[j] = j <= lane ? Lm[lane][j] : 0.0;
#pragma unroll
    for (int k = 0; k < CHOL_NB; k++) {
      const double akk = __shfl_sync(0xffffffffu, a[k], k);
      if (lane == 0 && k < nb && !(akk > 0.0)) *chol_fail += 1;
      const double rs = fast_rsqrt(fmin(fmax(akk, 1e-30), 1e30));
      rsd[k] = rs;
      const double l = lane >= k ? a[k] * rs : 0.0;
      a[k] = l;
#pragma unroll
      for (int j = k + 1; j < CHOL_NB; j++) { const double ljk = __shfl_sync(0xffffffffu, l, j); a[j] -= l * ljk; }
    }
    __syncwarp();
#pragma unroll
    for (int j = 0; j < CHOL_NB; j++) Lm[lane][j] = j <= lane ? a[j] : 0.0;
    __syncwarp();
    double z[CHOL_NB];
#pragma unroll
    for (int i = 0; i < CHOL_NB; i++) {
      double t0 = (i == lane) ? 1.0 : 0.0, t1 = 0.0, t2 = 0.0, t3 = 0.0;
#pragma unroll
      for (int m = 0; m < CHOL_NB; m += 4) {
        if (m < i) t0 -= Lm[i][m] * z[m];
        if (m + 1 < i) t1 -= Lm[i][m + 1] * z[m + 1];
        if (m + 2 < i) t2 -= Lm[i][m + 2] * z[m + 2];
        if (m + 3 < i) t3 -= Lm[i][m + 3] * z[m + 3];
      }
      z[i] = (i >= lane) ? ((t0 + t1) + (t2 + t3)) * rsd[i] : 0.0;
    }
#pragma unroll
    for (int i = 0; i < CHOL_NB; i++) Liv[i][lane] = z[i];
  }
  __syncthreads();
  double* Li = Linv_all + (size_t)(kb / CHOL_NB) * CHOL_NB * CHOL_NB;
  for (int o = tid; o < CHOL_NB * CHOL_NB; o += LM_THREADS) {
    const int i = o / CHOL_NB, j = o % CHOL_NB;
    if (i < nb && j <= i) S[(size_t)(kb + i) * n + kb + j] = Lm[i][j];
    Li[o] = Liv[i][j];
  }
  __syncthreads();
}
// ---- reduced solve, n <= 128: one CTA of 16 x 16 threads, matrix cyclically distributed in registers: thread (ty,tx) owns
// A[ty + 16 p][tx + 16 q].  After every 16 columns the register tile is ROTATED (a[p][q] <- a[p+1][q+1]) so that the active pivot
// block is always a[0][0] / column block q = 0: every register index on the pivot path is static, the path is ~45 instructions
// (round 1's switch over the column block: ~150).  The factor goes to shared memory column by column as it is produced.
template <int R>
__device__ __forceinline__ void chol_rot_body(int n, const double* Sg, const double* rhs, const double* gh, double reg, int* chol_fail, double* out, double* shm) {
  const int ld = n | 1;
  double* Lm = shm;                       // n x ld factor
  double* colbuf = Lm + (size_t)n * ld;   // n (+16 pad)
  double* invd = colbuf + n + 16;         // n
  double* piv = invd + n;                 // 2
  const int tid = threadIdx.x, ty = tid & 15, tx = tid >> 4;
  double a[R][R];
#pragma unroll
  for (int p = 0; p < R; p++)
#pragma unroll
    for (int q = 0; q < R; q++) {
      const int i = ty + 16 * p, j = tx + 16 * q;
      a[p][q] = (i < n && j < n) ? __ldcg(&Sg[(size_t)j * n + i]) + (i == j ? reg : 0.0) : 0.0;     // S is symmetric: coalesced read
    }
  __syncthreads();
  if (tid == 0) piv[0] = a[0][0];
  __syncthreads();
  const int nblk = (n + 15) >> 4;
  for (int kb = 0; kb < nblk; kb++) {
    const int k0 = 16 * kb;
    const int kend = min(16, n - k0);
    for (int kt = 0; kt < kend; kt++) {
      const int k = k0 + kt;
      if (tx == kt) {                      // the 16 threads that hold column k (block column 0 of the rotated tile)
        const double akk = piv[0];
        const double rs = fast_rsqrt(fmin(fmax(akk, 1e-30), 1e30));
        if (ty == kt) { invd[k] = rs; if (!(akk > 0.0)) *chol_fail += 1; }
#pragma unroll
        for (int p = 0; p < R; p++) {
          const int i = k0 + ty + 16 * p;
          if (i >= k && i < n) { const double lv = a[p][0] * rs; colbuf[i] = lv; Lm[i * ld + k] = lv; }
        }
      }
      __syncthreads();
      double ci[R], cj[R];
#pragma unroll
      for (int p = 0; p < R; p++) { const int i = k0 + ty + 16 * p; ci[p] = (i > k && i < n) ? colbuf[i] : 0.0; }
#pragma unroll
      for (int q = 0; q < R; q++) { const int j = k0 + tx + 16 * q; cj[q] = (j > k && j < n) ? colbuf[j] : 0.0; }
#pragma unroll
      for (int p = 0; p < R; p++)
#pragma unroll
        for (int q = 0; q < R; q++) a[p][q] -= ci[p] * cj[q];       // (also touches the unused upper triangle: harmless)
      // publish the next pivot: thread (kt+1, kt+1) of this block, or (0,0) of the next block (its a[1][1] before the rotation)
      if (kt + 1 < 16) { if (ty == kt + 1 && tx == kt + 1) piv[0] = a[0][0]; }
      else if (R > 1) { if (ty == 0 && tx == 0) piv[0] = a[R > 1 ? 1 : 0][R > 1 ? 1 : 0]; }
      __syncthreads();
    }
    // rotate: the next 16 x 16 pivot block moves to a[0][0]
#pragma unroll
    for (int p = 0; p < R; p++)
#pragma unroll
      for (int q = 0; q < R; q++) a[p][q] = (p + 1 < R && q + 1 < R) ? a[p + 1 < R ? p + 1 : p][q + 1 < R ? q + 1 : q] : 0.0;
  }
  __syncthreads();
  if (tid < 32) {
    constexpr int RS = (R * 16 + 31) / 32;       // rows per lane
    const int lane = tid;
    double bs[RS];
#pragma unroll
    for (int s2 = 0; s2 < RS; s2++) { const int i = lane + 32 * s2; bs[s2] = i < n ? __ldcg(&rhs[i]) + gh[i] : 0.0; }
    // forward: L y = b
#pragma unroll
    for (int s1 = 0; s1 < RS; s1++) {
      for (int kk = 0; kk < 32; kk++) {
        const int k = 32 * s1 + kk;
        if (k >= n) break;
        const double yk = __shfl_sync(0xffffffffu, bs[s1] * invd[k], kk);
        if (lane == kk) bs[s1] = yk;
#pragma unroll
        for (int s2 = s1; s2 < RS; s2++) { const int i = lane + 32 * s2; if (i > k && i < n) bs[s2] -= Lm[i * ld + k] * yk; }
      }
    }
    // backward: L^T x = y
#pragma unroll
    for (int s1 = RS - 1; s1 >= 0; s1--) {
      for (int kk = 31; kk >= 0; kk--) {
        const int k = 32 * s1 + kk;
        if (k >= n) continue;
        const double xk = __shfl_sync(0xffffffffu, bs[s1] * invd[k], kk);
        if (lane == kk) bs[s1] = xk;
#pragma unroll
        for (int s2 = 0; s2 <= s1; s2++) { const int i = lane + 32 * s2; if (i < k) bs[s2] -= Lm[k * ld + i] * xk; }
      }
    }
#pragma unroll
    for (int s2 = 0; s2 < RS; s2++) { const int i = lane + 32 * s2; if (i < n) out[i] = bs[s2]; }
  }
  __syncthreads();
}

// One 32x32 tile (ti >= tj) of the trailing update of panel p, with the panel solve folded in: X_i = A[rows_i, panel] L_pp^-T (a product
// with the inverted diagonal block -- lower triangular: output column c needs k <= c only), X_j likewise (the same thing on a diagonal
// tile), A[rows_i, cols_j] -= X_i X_j^T.  The tiles of block column 0 also store X_i as the finished factor -- TRANSPOSED, into the strict
// upper triangle (row kbp + k, column i): the lower triangle stays the working matrix that every other tile of this update still reads,
// the upper triangle collects L^T for the substitutions.  Every group of global loads is issued as a whole before anything is stored (the
// pointers are generic: a load cannot pass the store in front of it, and the L2 round trips would add up).  sh: 5 x 32 x 33 doubles.
__device__ __forceinline__ void chol_fused_tile(int n, int p, int ti, int tj, double* S, const double* Linv_all, double* sh) {
  constexpr int LD = CHOL_NB + 1, PER = CHOL_NB * CHOL_NB / LM_THREADS;
  double* Li = sh;
  double* Ai = sh + 1 * CHOL_NB * LD;
  double* Aj = sh + 2 * CHOL_NB * LD;
  double* Xi = sh + 3 * CHOL_NB * LD;
  double* Xj = sh + 4 * CHOL_NB * LD;
  const bool same = ti == tj;
  const int kbp = CHOL_NB * p, base = kbp + CHOL_NB;
  const int i0 = base + CHOL_NB * ti, j0 = base + CHOL_NB * tj;
  const double* Lg = Linv_all + (size_t)p * CHOL_NB * CHOL_NB;
  const int tid = threadIdx.x;
  __syncthreads();
  {
    double vl[PER], va[PER], vb[PER];
#pragma unroll
    for (int q = 0; q < PER; q++) {
      const int o = tid + LM_THREADS * q, r = o / CHOL_NB, c = o % CHOL_NB;
      vl[q] = __ldcg(&Lg[o]);
      va[q] = (i0 + r < n) ? __ldcg(&S[(size_t)(i0 + r) * n + kbp + c]) : 0.0;
      vb[q] = (!same && j0 + r < n) ? __ldcg(&S[(size_t)(j0 + r) * n + kbp + c]) : 0.0;
    }
#pragma unroll
    for (int q = 0; q < PER; q++) {
      const int o = tid + LM_THREADS * q, r = o / CHOL_NB, c = o % CHOL_NB;
      Li[r * LD + c] = vl[q]; Ai[r * LD + c] = va[q];
      if (!same) Aj[r * LD + c] = vb[q];
    }
  }
  __syncthreads();
  {
    // thread (r, cg) -> X[r][cg + 8 q], q = 0..3: interleaved columns (8 different shared-memory banks per row of the inverse) and balanced
    // triangular k loops: the k in [8 s, 8 s + 8) only reach the columns with q >= s
    const int r = tid >> 3, cg = tid & 7;
    double xi[4] = {0, 0, 0, 0}, xj[4] = {0, 0, 0, 0};
#pragma unroll
    for (int s4 = 0; s4 < 4; s4++) {
#pragma unroll
      for (int kk = 0; kk < 8; kk++) {
        const int k = 8 * s4 + kk;
        const double av = Ai[r * LD + k], bv = same ? 0.0 : Aj[r * LD + k];
#pragma unroll
        for (int q = s4; q < 4; q++) { const double l = Li[(cg + 8 * q) * LD + k]; xi[q] += av * l; xj[q] += bv * l; }      // X[i][j] = sum_k A[i][k] Linv[j][k]
      }
    }
#pragma unroll
    for (int q = 0; q < 4; q++) { Xi[r * LD + cg + 8 * q] = xi[q]; if (!same) Xj[r * LD + cg + 8 * q] = xj[q]; }
  }
  __syncthreads();
  if (same) Xj = Xi;
  if (tj == 0)
    for (int o = tid; o < CHOL_NB * CHOL_NB; o += LM_THREADS) {      // L^T into the upper triangle, coalesced over the factor's rows
      const int c = o >> 5, r = o & 31;
      if (i0 + r < n) S[(size_t)(kbp + c) * n + i0 + r] = Xi[r * LD + c];
    }
  {
    const int tx = tid & 15, ty = tid >> 4;
    // the tile's old values: in flight while the product runs (last written by another CTA in the previous panel: from L2)
    double old[2][2];
#pragma unroll
    for (int pp = 0; pp < 2; pp++)
#pragma unroll
      for (int q = 0; q < 2; q++) {
        const int i = i0 + ty + 16 * pp, j = j0 + tx + 16 * q;
        old[pp][q] = (i < n && j < n && j <= i) ? __ldcg(&S[(size_t)i * n + j]) : 0.0;
      }
    double acc[2][2] = {{0, 0}, {0, 0}};
#pragma unroll 8
    for (int k = 0; k < CHOL_NB; k++) {
      const double a0 = Xi[ty * LD + k], a1 = Xi[(ty + 16) * LD + k], b0 = Xj[tx * LD + k], b1 = Xj[(tx + 16) * LD + k];
      acc[0][0] += a0 * b0; acc[0][1] += a0 * b1; acc[1][0] += a1 * b0; acc[1][1] += a1 * b1;
    }
#pragma unroll
    for (int pp = 0; pp < 2; pp++)
#pragma unroll
      for (int q = 0; q < 2; q++) {
        const int i = i0 + ty + 16 * pp, j = j0 + tx + 16 * q;
        if (i < n && j < n && j <= i) S[(size_t)i * n + j] = old[pp][q] - acc[pp][q];
      }
  }
}

constexpr int SUBST_HALF = 16, SUBST_UN = 8;
// Both substitutions by one CTA with the factor in global memory (lower = working matrix, strict upper = L^T collected by the tiles) and
// the inverted diagonal blocks.  What a block needs from the factor does not depend on the solution, so nothing of it may sit on the
// critical path behind an L2 round trip more than once: the inverted diagonal block of the NEXT block is fetched while this one is worked
// on (shared memory, double buffered), and the block's panel of L^T -- rows 32 j .. 32 j + 31, each contiguous -- is read with all the
// loads of a thread in flight at once: forward in axpy form (thread = column i: b_i -= sum_k L^T[k][i] y_k, 32 loads per column, the
// next block's rows first), backward over the SAME panels in dot form (thread = (rows k, k + 16; column slice): 16 loads in flight, the 16
// slices of a row reduced by shuffles).  Fixed order everywhere.  Slower forms this replaced: two dependent L2 round trips
// per block and direction with 8-deep load batches; the panels through a 4-stage ring of bulk asynchronous copies (16 requests of 2 KB
// per stage), where a stage cost what the copy unit takes for 16 requests.
__host__ __device__ inline size_t subst_smem_doubles(int n) {
  return (size_t)((n + CHOL_NB - 1) / CHOL_NB) * CHOL_NB + 2 * CHOL_NB * (CHOL_NB + 1) + 64;
}
__device__ __noinline__ void chol_substitute_body(int n, const double* L, const double* Linv_all, const double* rhs, const double* gh, double* out, double* sh) {
  constexpr int LVS = CHOL_NB + 1;
  const int tid = threadIdx.x;
  const int nblk = (n + CHOL_NB - 1) / CHOL_NB, npad = nblk * CHOL_NB;
  double* bsh = sh;                                   // [npad]  b -> y -> x
  double* Lv = bsh + npad;                            // [2][32][33]  inverted diagonal blocks, double buffered
  double* tv = Lv + 2 * CHOL_NB * LVS;                // [64]  y of the block in progress | reduced dots
  __syncthreads();
  for (int i = tid; i < npad; i += LM_THREADS) bsh[i] = i < n ? __ldcg(&rhs[i]) + gh[i] : 0.0;
  auto load_linv = [&](int blk, double (&r)[4]) {
    const double* Li = Linv_all + (size_t)blk * CHOL_NB * CHOL_NB;
#pragma unroll
    for (int q = 0; q < 4; q++) r[q] = __ldcg(&Li[tid + LM_THREADS * q]);
  };
  auto store_linv = [&](int blk, const double (&r)[4]) {
    double* dst = Lv + (size_t)(blk & 1) * CHOL_NB * LVS;
#pragma unroll
    for (int q = 0; q < 4; q++) { const int o = tid + LM_THREADS * q; dst[(o >> 5) * LVS + (o & 31)] = r[q]; }
  };
  double lr[4];
  load_linv(0, lr); store_linv(0, lr);
  __syncthreads();
  // ---- forward: L y = b
  for (int blk = 0; blk < nblk; blk++) {
    const int kb = CHOL_NB * blk;
    const bool has_next = blk + 1 < nblk;
    if (has_next) load_linv(blk + 1, lr);             // in flight while this block is worked on
    const double* Lb = Lv + (size_t)(blk & 1) * CHOL_NB * LVS;
    if (tid < CHOL_NB) {
      double a0 = 0.0, a1 = 0.0, a2 = 0.0, a3 = 0.0;
#pragma unroll
      for (int k = 0; k < CHOL_NB; k += 4) {
        a0 += Lb[tid * LVS + k] * bsh[kb + k]; a1 += Lb[tid * LVS + k + 1] * bsh[kb + k + 1];
        a2 += Lb[tid * LVS + k + 2] * bsh[kb + k + 2]; a3 += Lb[tid * LVS + k + 3] * bsh[kb + k + 3];
      }
      tv[tid] = (a0 + a1) + (a2 + a3);
    }
    __syncthreads();
    if (tid < CHOL_NB) bsh[kb + tid] = tv[tid];
    for (int i = kb + CHOL_NB + tid; i < n; i += LM_THREADS) {
      const double* col = L + (size_t)kb * n + i;     // L^T[kb + k][i], k = 0..31: coalesced over i
      double l[CHOL_NB];
#pragma unroll
      for (int k = 0; k < CHOL_NB; k++) l[k] = __ldcg(col + (size_t)k * n);
      double a0 = 0.0, a1 = 0.0, a2 = 0.0, a3 = 0.0;
#pragma unroll
      for (int k = 0; k < CHOL_NB; k += 4) { a0 += l[k] * tv[k]; a1 += l[k + 1] * tv[k + 1]; a2 += l[k + 2] * tv[k + 2]; a3 += l[k + 3] * tv[k + 3]; }
      bsh[i] -= (a0 + a1) + (a2 + a3);
    }
    if (has_next) store_linv(blk + 1, lr);
    __syncthreads();
  }
  // ---- backward: L^T x = y.  The last block's inverse is still in its buffer.
  const int kk = tid >> 4, sl = tid & 15;
  for (int blk = nblk - 1; blk >= 0; blk--) {
    const int kb = CHOL_NB * blk;
    const bool has_next = blk > 0;
    if (has_next) load_linv(blk - 1, lr);
    const double* Lb = Lv + (size_t)(blk & 1) * CHOL_NB * LVS;
    // t_k = sum_{i >= kb + 32} L^T[kb + k][i] x_i: thread (kk, sl) -> rows kk, kk + 16, columns == sl (mod 16)
    double p0 = 0.0, p1 = 0.0;
    {
      const double* r0 = L + (size_t)(kb + kk) * n, *r1 = r0 + (size_t)SUBST_HALF * n;
      for (int i0 = kb + CHOL_NB + sl; i0 < n; i0 += 16 * SUBST_UN) {
        double l0[SUBST_UN], l1[SUBST_UN];
#pragma unroll
        for (int u = 0; u < SUBST_UN; u++) { const int i = i0 + 16 * u; const bool on = i < n; l0[u] = on ? __ldcg(r0 + i) : 0.0; l1[u] = on ? __ldcg(r1 + i) : 0.0; }
#pragma unroll
        for (int u = 0; u < SUBST_UN; u++) { const int i = i0 + 16 * u; const double xv = i < n ? bsh[i] : 0.0; p0 += l0[u] * xv; p1 += l1[u] * xv; }
      }
    }
#pragma unroll
    for (int o = 8; o > 0; o >>= 1) { p0 += __shfl_xor_sync(0xffffffffu, p0, o); p1 += __shfl_xor_sync(0xffffffffu, p1, o); }
    if (sl == 0) { tv[kk] = p0; tv[SUBST_HALF + kk] = p1; }
    __syncthreads();
    if (tid < CHOL_NB) tv[32 + tid] = bsh[kb + tid] - tv[tid];
    __syncthreads();
    if (tid < CHOL_NB) {
      double a0 = 0.0, a1 = 0.0, a2 = 0.0, a3 = 0.0;
#pragma unroll
      for (int k = 0; k < CHOL_NB; k += 4) {
        a0 += Lb[k * LVS + tid] * tv[32 + k]; a1 += Lb[(k + 1) * LVS + tid] * tv[32 + k + 1];
        a2 += Lb[(k + 2) * LVS + tid] * tv[32 + k + 2]; a3 += Lb[(k + 3) * LVS + tid] * tv[32 + k + 3];
      }
      bsh[kb + tid] = (a0 + a1) + (a2 + a3);
    }
    if (has_next) store_linv(blk - 1, lr);
    __syncthreads();
  }
  for (int i = tid; i < n; i += LM_THREADS) out[i] = bsh[i];
  __syncthreads();
}

// shared memory of k_lm in doubles
__host__ __device__ inline size_t lm_smem_doubles(int n_s, int fb) {
  const size_t small = n_s <= CHOL_SMALL_MAX ? (size_t)n_s * (n_s | 1) + 2 * (size_t)n_s + 32 : 0;
  const size_t big = n_s > CHOL_SMALL_MAX ? subst_smem_doubles(n_s) : 0;
  const size_t syrk = (size_t)SYRK_STAGES * 2 * SYRK_K * SYRK_TILE;
  const size_t chol_tiles = 5 * (size_t)CHOL_NB * (CHOL_NB + 1) + 3 * CHOL_NB;
  const size_t frames = (size_t)LM_WARPS * (12 * 12 + 12);
  size_t m = small;
  if (big > m) m = big;
  if (syrk > m) m = syrk;
  if (chol_tiles > m) m = chol_tiles;
  if (frames > m) m = frames;
  return m + 64;
}

// ---------------------------------------------------------------- the kernel
template <int FB>
__global__ void __launch_bounds__(LM_THREADS, 1)
k_lm(LmArgs a) {
  extern __shared__ double ksm[];
  __shared__ SolverState S;
  __shared__ double sm[32];
  __shared__ int xerr, chol_fail_s;
  __shared__ __align__(8) unsigned long long sbar[SYRK_STAGES];      // mbarriers of the SYRK operand pipeline
  unsigned sphases = 0;                                               // their phase parities (same in every thread)
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int n = a.n, n_s = a.n_s;
  const int F = a.P.motion_on ? a.F : 0;              // frames with a free block
  const int nblk = gridDim.x;
  const int gthread = blockIdx.x * LM_THREADS + tid, gstride = nblk * LM_THREADS;
  const int gwarp = blockIdx.x * LM_WARPS + warp, gwarps = nblk * LM_WARPS;
  const bool multi = a.peer.world > 1;
  const bool writer = blockIdx.x == 0 && tid == 0;
  double* work = ksm + 64;

  if (tid == 0) { S = *a.st; xerr = 0; chol_fail_s = 0; for (int q = 0; q < SYRK_STAGES; q++) mbar_init(&sbar[q], 1); fence_barrier_init(); }
  if (a.prof && blockIdx.x == 0 && tid == 0) a.prof[0] = 0;
#ifdef MCBA_SIMT_BUILD
#define LMPH(ID_) simt::set_mark(ID_);
#else
#define LMPH(ID_) if (a.prof && blockIdx.x == 0 && tid == 0) { unsigned long long t_; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_)); a.prof[ID_] = t_; }
#endif
  __syncthreads();
  if (S.done) {
    if (writer && a.use_cond) cudaGraphSetConditional((cudaGraphConditionalHandle)a.cond_handle, 0);
    return;
  }
  unsigned long long xseq = 0;
  if (multi) xseq = *a.peer.seq;                       // exchanges done so far (every CTA reads the same value: written at the end of the previous launch)

  auto log_row = [&](int it, int nfev, double cost, double red, double step, double opt) {
    if (writer && S.nlog < a.log_cap) a.log[S.nlog] = mcba_log_row{it, nfev, cost, red, step, opt};
    if (tid == 0) S.nlog += 1;
  };

  // ------------------------------------------------------------------------------------------ phase A: the pending trial
  LMPH(1)
  bool need_solve = true;
  double first_cost = 0.0;                              // several GPUs: cost of the first linearisation summed over the ranks
  if (S.pending) {
    double cost_new = sum_records(a.frame_cost, a.F, 1, 0, sm);
    double s2f = sum_records(a.part_step, S.step_parts, 2, 0, sm);
    double x2f = sum_records(a.part_step, S.step_parts, 2, 1, sm);
    if (multi) {
      // one exchange: trial cost and step norms (frame parts) of all ranks, and -- the trial is linearised speculatively -- the shared
      // gradient / diagonal / cost of its normal equations, which the next iteration starts from if the step is accepted
      if (writer) { a.part_quad[0] = cost_new; a.part_quad[1] = s2f; a.part_quad[2] = x2f; }
      grid_barrier(a.bar, nblk);
      XSeg seg[3] = {{a.part_quad, 3, 0}, {const_cast<double*>(a.g), n_s, 0}, {a.S, n_s, 0}};
      // diag(H_ss) travels in the first n_s entries of S (S is rebuilt in phase D)
      for (int i = gthread; i < n_s; i += gstride) a.S[i] = a.Hss[(size_t)i * n_s + i];
      grid_barrier(a.bar, nblk);
      exchange(a, seg, 3, ++xseq, &xerr);
      cost_new = __ldcg(&a.part_quad[0]); s2f = __ldcg(&a.part_quad[1]); x2f = __ldcg(&a.part_quad[2]);
    }
    if (tid == 0) accept_compute(&S, cost_new, S.step2_s, s2f, S.xn2_s, x2f);
    __syncthreads();
    const bool accepted = S.accepted != 0, may_retry = S.status == -99 && S.nfev < S.max_nfev;
    __syncthreads();                                    // thread 0 updates S below: every thread has its copy of the decision first
    if (accepted) {
      // x = x_new ; cost = cost_new ; J = jac(x)  (trf.py): the trial state becomes the current one
      for (int i = gthread; i < n; i += gstride) a.x[i] = a.x_new[i];
      // (the fixed blocks of the trial state equal the current ones: the solve starts from a copy, make_trial_item copies them)
      for (int i = gthread; i < a.state_len; i += gstride) a.P.cam_rt[i] = a.trial[i];
      if (tid == 0) {
        S.cost = S.cost_new; S.njev += 1; S.last_reduction = S.actual_reduction; S.last_step_norm = S.step_norm;
        S.iteration += 1; S.accepted = 0; S.pending = 0;
      }
    } else if (may_retry) {
      need_solve = false;                                 // shrink the radius and try again from the same model (trf.py inner loop)
    } else {
      // out of evaluations, or a termination test fired on a step that did not reduce the cost: the loop ends at the unchanged x
      if (tid == 0) { S.iteration += 1; S.last_reduction = 0.0; S.last_step_norm = 0.0; S.done = 1; S.pending = 0; }
      __syncthreads();
      log_row(S.iteration, S.nfev, S.cost, 0.0, 0.0, S.g_norm);
      __syncthreads();
      if (writer) { *a.st = S; if (multi) *a.peer.seq = xseq; if (a.use_cond) cudaGraphSetConditional((cudaGraphConditionalHandle)a.cond_handle, 0); }
      return;
    }
    __syncthreads();
  } else if (multi) {
    // first linearisation: shared gradient, diagonal and cost of all ranks
    for (int i = gthread; i < n_s; i += gstride) a.S[i] = a.Hss[(size_t)i * n_s + i];
    if (writer) a.part_quad[0] = *a.lin_cost;
    grid_barrier(a.bar, nblk);
    XSeg seg[3] = {{a.part_quad, 1, 0}, {const_cast<double*>(a.g), n_s, 0}, {a.S, n_s, 0}};
    exchange(a, seg, 3, ++xseq, &xerr);
    first_cost = __ldcg(&a.part_quad[0]);
  }

  if (need_solve) {
    LMPH(2)
    // ---------------------------------------------------------------------------------------- phase B: scaling, g_h, norms
    {
      double gh2s = 0, gh2f = 0, gms = 0, gmf = 0, xs2s = 0, xs2f = 0;
      const int first = S.first_scale;
      for (int i = gthread; i < n; i += gstride) {
        double hd;
        if (i < n_s) hd = multi ? __ldcg(&a.S[i]) : a.Hss[(size_t)i * n_s + i];
        else { const int f = (i - n_s) / FB, j = (i - n_s) % FB; hd = a.Hff[(size_t)f * FB * FB + j * (FB + 1)]; }
        const double nrm = sqrt(fmax(hd, 0.0));
        double si;
        if (first) si = (nrm == 0.0) ? 1.0 : nrm; else si = fmax(nrm, a.sinv[i]);
        a.sinv[i] = si;
        const double di = 1.0 / si;
        a.d[i] = di;
        const double gi = a.g[i], ghi = di * gi, xs = a.x[i] * si;
        a.gh[i] = ghi;
        if (i < n_s) { gh2s += ghi * ghi; gms = fmax(gms, fabs(gi)); xs2s += xs * xs; }
        else { gh2f += ghi * ghi; gmf = fmax(gmf, fabs(gi)); xs2f += xs * xs; }
      }
      const double r0 = block_sum_all(gh2s, sm), r1 = block_sum_all(gh2f, sm), r2 = block_max_all(gms, sm), r3 = block_max_all(gmf, sm);
      const double r4 = block_sum_all(xs2s, sm), r5 = block_sum_all(xs2f, sm);
      if (tid == 0) { double* q = a.part_scale + (size_t)blockIdx.x * 6; q[0] = r0; q[1] = r1; q[2] = r2; q[3] = r3; q[4] = r4; q[5] = r5; }
    }
    grid_barrier(a.bar, nblk);
    {
      double gh2s = sum_records(a.part_scale, nblk, 6, 0, sm), gh2f = sum_records(a.part_scale, nblk, 6, 1, sm);
      double gms = max_records(a.part_scale, nblk, 6, 2, sm), gmf = max_records(a.part_scale, nblk, 6, 3, sm);
      double xs2s = sum_records(a.part_scale, nblk, 6, 4, sm), xs2f = sum_records(a.part_scale, nblk, 6, 5, sm);
      double lin_cost = __ldcg(a.lin_cost);
      if (multi) {
        // the shared entries are replicated (identical on every rank after the first exchange): only the frame parts travel
        if (writer) { a.part_quad[0] = gh2f; a.part_quad[1] = xs2f; a.part_quad[2] = gmf; }
        grid_barrier(a.bar, nblk);
        XSeg seg[2] = {{a.part_quad, 2, 0}, {a.part_quad + 2, 1, 1}};
        exchange(a, seg, 2, ++xseq, &xerr);
        gh2f = __ldcg(&a.part_quad[0]); xs2f = __ldcg(&a.part_quad[1]); gmf = __ldcg(&a.part_quad[2]);
      }
      if (tid == 0) {
        begin_iteration(&S, gh2s, gh2f, gms, gmf, xs2s, xs2f, multi ? first_cost : lin_cost);     // the cost is read on the first call only
        if (!isfinite(S.cost)) { S.done = 1; S.status = -2; }          // non-finite residuals at the initial point (scipy raises ValueError)
      }
      __syncthreads();
      log_row(S.iteration, S.nfev, S.cost, S.iteration == 0 ? NAN : S.last_reduction, S.iteration == 0 ? NAN : S.last_step_norm, S.g_norm);
      __syncthreads();
      if (S.done) {
        if (writer) { *a.st = S; if (multi) *a.peer.seq = xseq; if (a.use_cond) cudaGraphSetConditional((cudaGraphConditionalHandle)a.cond_handle, 0); }
        return;
      }
    }
    // ---------------------------------------------------------------------------------------- phase C: g_h^T A g_h -> reg
    const int nsh = n_s;                                           // records of the shared rows (one per row)
    auto quad_pass = [&](const double* u, const double* v, int two, double* partial /*[F + n_s][5]*/) {
      for (int f = gwarp; f < F; f += gwarps) {
        const double* Wf = a.W + (size_t)f * n_s * FB;
        double tu[FB], tv[FB];
#pragma unroll
        for (int j = 0; j < FB; j++) { tu[j] = 0.0; tv[j] = 0.0; }
        // a lane's FB doubles of a row are 16-byte aligned (FB even): double2 loads, four rows in flight per lane
#pragma unroll 4
        for (int s = lane; s < n_s; s += 32) {
          const double us = a.d[s] * u[s], vs = two ? a.d[s] * v[s] : 0.0;
          const double2* w2 = reinterpret_cast<const double2*>(Wf + (size_t)s * FB);
#pragma unroll
          for (int j = 0; j < FB / 2; j++) { const double2 w = w2[j]; tu[2 * j] += w.x * us; tv[2 * j] += w.x * vs; tu[2 * j + 1] += w.y * us; tv[2 * j + 1] += w.y * vs; }
        }
#pragma unroll
        for (int j = 0; j < FB; j++) {
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) { tu[j] += __shfl_xor_sync(0xffffffffu, tu[j], o); tv[j] += __shfl_xor_sync(0xffffffffu, tv[j], o); }
        }
        if (lane == 0) {
          double uf[FB], vf[FB], uu = 0, uv = 0, vv = 0, dt = 0, g2 = 0;
#pragma unroll
          for (int j = 0; j < FB; j++) { const int i = n_s + FB * f + j; uf[j] = a.d[i] * u[i]; vf[j] = two ? a.d[i] * v[i] : 0.0; if (two) { dt += u[i] * v[i]; g2 += v[i] * v[i]; } }
          const double* H = a.Hff + (size_t)f * FB * FB;
#pragma unroll
          for (int i = 0; i < FB; i++) {
            double hu = 0, hv = 0;
#pragma unroll
            for (int j = 0; j < FB; j++) { hu += H[i * FB + j] * uf[j]; hv += H[i * FB + j] * vf[j]; }
            uu += uf[i] * (hu + 2.0 * tu[i]);
            uv += uf[i] * hv + uf[i] * tv[i] + vf[i] * tu[i];
            vv += vf[i] * (hv + 2.0 * tv[i]);
          }
          double* q = partial + (size_t)f * 5;
          q[0] = uu; q[1] = uv; q[2] = vv; q[3] = dt; q[4] = g2;
        }
      }
      // shared rows: a warp per row of H_ss (contiguous: coalesced), one record per row.  (A thread per COLUMN walking all rows had only
      // ceil(n_s / 256) CTAs at work on a serial chain of n_s L2 round trips: most of phase C at n_s = 286 and 1030.)
      for (int j = gwarp; j < n_s; j += gwarps) {
        const double* Hr = a.Hss + (size_t)j * n_s;
        double hu = 0.0, hv = 0.0;
#pragma unroll 4
        for (int i = lane; i < n_s; i += 32) {
          const double h = Hr[i], di = a.d[i];
          hu += h * (di * u[i]);
          if (two) hv += h * (di * v[i]);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) { hu += __shfl_xor_sync(0xffffffffu, hu, o); hv += __shfl_xor_sync(0xffffffffu, hv, o); }
        if (lane == 0) {
          const double uj = a.d[j] * u[j], vj = two ? a.d[j] * v[j] : 0.0;
          double* q = partial + (size_t)(F + j) * 5;
          q[0] = uj * hu; q[1] = uj * hv; q[2] = vj * hv; q[3] = two ? u[j] * v[j] : 0.0; q[4] = two ? v[j] * v[j] : 0.0;
        }
      }
    };
    LMPH(3)
    quad_pass(a.gh, a.gh, 0, a.part_quad + 8);
    grid_barrier(a.bar, nblk);
    {
      double agg = sum_records(a.part_quad + 8, F + nsh, 5, 0, sm);
      if (multi) {
        // H_ss is this rank's local part: its quadratic form sums over the ranks like the frame parts
        if (writer) a.part_quad[0] = agg;
        grid_barrier(a.bar, nblk);
        XSeg seg[1] = {{a.part_quad, 1, 0}};
        exchange(a, seg, 1, ++xseq, &xerr);
        agg = __ldcg(&a.part_quad[0]);
      }
      if (tid == 0) { reg_compute(&S, agg); S.agg = agg; }
      __syncthreads();
    }
    LMPH(4)
    const double reg = S.reg;
    // ---------------------------------------------------------------------------------------- phase D: frames out, S in
    for (size_t idx = gthread; idx < (size_t)n_s * n_s; idx += gstride) {
      const int i = idx / n_s, j = idx % n_s;
      a.S[idx] = a.d[i] * a.d[j] * a.Hss[idx];
    }
    if (F > 0) {
      double* Lw = work + (size_t)warp * (FB * FB + FB);
      for (int f = gwarp; f < F; f += gwarps) schur_frame<FB>(a, f, reg, lane, Lw);
    }
    grid_barrier(a.bar, nblk);
    // ---------------------------------------------------------------------------------------- phase E: S -= sum_f Y_f Y_f^T
    LMPH(5)
    if (F > 0 && n_s > 0) {
      const int tiles = (n_s + SYRK_TILE - 1) / SYRK_TILE;
      const int npair = tiles * (tiles + 1) / 2;
      for (int vb = blockIdx.x; vb < npair * a.syrk_chunks; vb += nblk) {
        const int chunk = vb / npair; int pr = vb % npair;
        int ti = 0; while (pr >= tiles - ti) { pr -= tiles - ti; ti++; }
        const int tj = ti + pr;
        syrk_tile<FB>(a, ti, tj, chunk, work, sbar, sphases);
      }
      grid_barrier(a.bar, nblk);
      // fixed-order sum over the frame chunks; tiles hold the upper triangle (ti <= tj), S is kept full
      for (size_t idx = gthread; idx < (size_t)n_s * n_s; idx += gstride) {
        const int i = idx / n_s, j = idx % n_s;
        const int ii = min(i, j), jj = max(i, j);
        // inside a diagonal tile both triangles were computed; everywhere else take the (ii, jj) entry
        double s = 0.0;
        for (int c = 0; c < a.syrk_chunks; c++) s += __ldcg(&a.Spart[(size_t)c * n_s * n_s + (size_t)ii * n_s + jj]);
        a.S[idx] -= s;
      }
      for (int i = gthread; i < n_s; i += gstride) {
        double s = 0.0;
        for (int c = 0; c < a.syrk_chunks; c++) s += __ldcg(&a.rpart[(size_t)c * n_s + i]);
        a.rhs[i] = -s;
      }
    } else {
      for (int i = gthread; i < n_s; i += gstride) a.rhs[i] = 0.0;
    }
    grid_barrier(a.bar, nblk);
    if (multi && n_s > 0) {
      XSeg seg[2] = {{a.S, n_s * n_s, 0}, {a.rhs, n_s, 0}};
      exchange(a, seg, 2, ++xseq, &xerr);
    }
    // ---------------------------------------------------------------------------------------- phase F: reduced solve
    LMPH(6)
    if (n_s > 0) {
      if (n_s <= CHOL_SMALL_MAX) {
        if (blockIdx.x == 0) {
          const int R = (n_s + 15) / 16;
#define CS(RR) case RR: chol_rot_body<RR>(n_s, a.S, a.rhs, a.gh, reg, &chol_fail_s, a.gn, work); break;
          switch (R) { CS(1) CS(2) CS(3) CS(4) CS(5) CS(6) CS(7) CS(8) }
#undef CS
        }
      } else {
        for (int i = gthread; i < n_s; i += gstride) a.S[(size_t)i * n_s + i] += reg;
        grid_barrier(a.bar, nblk);
        // one barrier per panel: CTA 0 finishes the next diagonal block's tile of the previous trailing update first and factors it
        // (look-ahead) while the other CTAs work off the rest of that update
        const int npan = (n_s + CHOL_NB - 1) / CHOL_NB;
        for (int b = 0; b < npan; b++) {
          const int kb = CHOL_NB * b;
          const int rem = b > 0 ? n_s - kb : 0;                       // rows of the trailing matrix of panel b-1
          const int t = (rem + CHOL_NB - 1) / CHOL_NB, ntile = t * (t + 1) / 2;
          if (blockIdx.x == 0) {
            if (b > 0) chol_fused_tile(n_s, b - 1, 0, 0, a.S, a.Linv, work);
            chol_diag_warp_body(n_s, kb, a.S, a.Linv, &chol_fail_s, work);
          }
          if (b > 0) {
            const int first = nblk > 1 ? (int)blockIdx.x - 1 : 0, step = nblk > 1 ? nblk - 1 : 1;
            if (nblk == 1 || blockIdx.x > 0)
              for (int vb = 1 + first; vb < ntile; vb += step) {
                int ti = 0, pr = vb; while (pr > ti) { pr -= ti + 1; ti++; }        // lower triangle: ti >= tj = pr
                chol_fused_tile(n_s, b - 1, ti, pr, a.S, a.Linv, work);
              }
          }
          grid_barrier(a.bar, nblk);
        }
        LMPH(11)
        if (blockIdx.x == 0) {
          chol_substitute_body(n_s, a.S, a.Linv, a.rhs, a.gh, a.gn, work);
        }
        LMPH(12)
      }
    }
    grid_barrier(a.bar, nblk);
    // ---------------------------------------------------------------------------------------- phase G: back-substitution + subspace forms
    LMPH(7)
    for (int f = gwarp; f < F; f += gwarps) {
      const double* Yf = a.Y + (size_t)f * SYRK_TILE * FB;
      const size_t ytile = (size_t)a.F * SYRK_TILE * FB;
      double t[FB];
#pragma unroll
      for (int k = 0; k < FB; k++) t[k] = 0.0;
#pragma unroll 4
      for (int s = lane; s < n_s; s += 32) {
        const double ps = __ldcg(&a.gn[s]);
        const double2* y2 = reinterpret_cast<const double2*>(Yf + (size_t)(s >> 5) * ytile + (size_t)(s & 31) * FB);
#pragma unroll
        for (int k = 0; k < FB / 2; k++) { const double2 y = y2[k]; t[2 * k] += y.x * ps; t[2 * k + 1] += y.y * ps; }
      }
#pragma unroll
      for (int k = 0; k < FB; k++) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) t[k] += __shfl_xor_sync(0xffffffffu, t[k], o);
      }
      if (lane == 0) {
        const double* L = a.Lf + (size_t)f * FB * FB;
        double y[FB];
#pragma unroll
        for (int i = 0; i < FB; i++) y[i] = a.zf[(size_t)f * FB + i] - t[i];
#pragma unroll
        for (int i = FB - 1; i >= 0; i--) {
          double v = y[i];
#pragma unroll
          for (int k = 0; k < FB; k++) if (k > i) v -= L[k * FB + i] * y[k];
          y[i] = v * L[i * FB + i];                            // the stored diagonal is 1 / L_ii
        }
#pragma unroll
        for (int i = 0; i < FB; i++) a.gn[n_s + FB * f + i] = y[i];
      }
      __syncwarp();
    }
    __syncthreads();      // a warp's gn_f stores are read by the same warp below (same frame -> same warp: gwarp stride is identical)
    LMPH(8)
    quad_pass(a.gh, a.gn, 1, a.part_quad + 8);
    grid_barrier(a.bar, nblk);
    {
      double agn = sum_records(a.part_quad + 8, F + nsh, 5, 1, sm), ann = sum_records(a.part_quad + 8, F + nsh, 5, 2, sm);
      double dtf = sum_records(a.part_quad + 8, F, 5, 3, sm), g2f = sum_records(a.part_quad + 8, F, 5, 4, sm);
      const double dts = sum_records(a.part_quad + 8 + (size_t)F * 5, nsh, 5, 3, sm), g2s = sum_records(a.part_quad + 8 + (size_t)F * 5, nsh, 5, 4, sm);
      if (multi) {
        if (writer) { a.part_quad[0] = agn; a.part_quad[1] = ann; a.part_quad[2] = dtf; a.part_quad[3] = g2f; }
        grid_barrier(a.bar, nblk);
        XSeg seg[1] = {{a.part_quad, 4, 0}};
        exchange(a, seg, 1, ++xseq, &xerr);
        agn = __ldcg(&a.part_quad[0]); ann = __ldcg(&a.part_quad[1]); dtf = __ldcg(&a.part_quad[2]); g2f = __ldcg(&a.part_quad[3]);
      }
      if (tid == 0) subspace_compute(&S, S.agg, agn, ann, dts, dtf, g2s, g2f);
      __syncthreads();
    }
  }

  // ------------------------------------------------------------------------------------------ phase I: step and trial state
  LMPH(9)
  if (tid == 0) tr_step_compute(&S);
  __syncthreads();
  {
    const double al = S.alpha, be = S.beta;
    double s2f = 0, x2f = 0;
    for (int i = gthread; i < n; i += gstride) {
      const double stp = a.d[i] * (al * a.gh[i] + be * __ldcg(&a.gn[i]));
      const double xi = a.x[i];
      a.x_new[i] = xi + stp;
      if (i >= n_s) { s2f += stp * stp; x2f += xi * xi; }
    }
    // the shared entries are few (n_s): every CTA sums them itself (replicated); the frame parts go to per-CTA records for the next launch
    double ss = 0, xs = 0;
    for (int i = tid; i < n_s; i += LM_THREADS) {
      const double stp = a.d[i] * (al * a.gh[i] + be * __ldcg(&a.gn[i]));
      const double xi = __ldcg(&a.x[i]);                   // copied by another CTA in phase A of this launch
      ss += stp * stp; xs += xi * xi;
    }
    ss = block_sum_all(ss, sm); xs = block_sum_all(xs, sm);
    const double r0 = block_sum_all(s2f, sm), r1 = block_sum_all(x2f, sm);
    if (tid == 0) { a.part_step[(size_t)blockIdx.x * 2] = r0; a.part_step[(size_t)blockIdx.x * 2 + 1] = r1; S.step2_s = ss; S.xn2_s = xs; S.step_parts = nblk; S.pending = 1; }
  }
  grid_barrier(a.bar, nblk);
  for (int i = gthread; i < a.n_items; i += gstride)
    make_trial_item(a.P, a.x_new, a.trial, i);
  __syncthreads();
  LMPH(10)
  if (writer) {
    if (xerr) { S.done = 1; S.status = -3; }
    S.chol_fail += chol_fail_s;
    *a.st = S;
    if (multi) *a.peer.seq = xseq;
    if (a.use_cond) cudaGraphSetConditional((cudaGraphConditionalHandle)a.cond_handle, S.done ? 0 : 1);
  }
}

}  // namespace mcba
