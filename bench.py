#!/usr/bin/env python
"""bench.py — reprojection residuals/sec and LM iterations/sec of the bundle-adjustment hot path.

  python bench.py [--gpus N] [--steps K] [--warmup W] [--workload cfg4] [--impl ours|reference] [--dump-outputs DIR]

One "step" = one full `bundle_adjust()` (calibration.py:199-212 semantics: ftol=1e-4, max_nfev=100, linear loss) over one
synthetic scene of the BASELINE.json configuration `--workload`.  Default workload at EVERY N: cfg4 = configs[3] (16 cameras x
1000 frames x 5 cube boards, 5.5 M corners) -- the largest configuration that fits one GPU and the one BASELINE names for 2/4/8
GPUs; with N > 1 the SAME scene is sharded by frame (strong scaling), and rank 0 also solves it alone and asserts that the sharded
solve ends at the same cost.  Secondary blocks in the same JSON line: cfg2, cfg3 and cfg5 at N = 1, weak scaling (cfg2 per GPU) at N > 1.
Metric (both arms, same definition):
    residuals/s = N_corners * (nfev + njev) / time      1 residual = one inlier corner (2 scalars),
    nfev/njev = cost and Jacobian evaluations as the solver reports them (scipy's res.nfev/res.njev for the reference arm; its
    finite-difference sub-evaluations are NOT counted, they are an artefact of its Jacobian).
`value`  : solves timed on the device with the packed problem already resident in HBM (CUDA events on the solver's stream).
`e2e`    : the same through the public API `Calibration.bundle_adjust()` from pinned host numpy buffers: packing, H2D, solve, D2H of
           the solved parameters all inside the timed region (wall clock, device synchronised).
`--impl reference` times the reference's CPU path on the host cores on a bounded frame-subsample of the same workload, through its
numpy + scipy restatement oracle/ba_oracle.py (the identical scipy.optimize.least_squares call).
`--dump-outputs DIR` writes what the last timed device-resident solve of the main workload computed, as float64 .npy files: the solved
parameters (cam_rt, board_rt, frame_rt, intrinsics: what Engine.get_params returns) and solve.npy = [cost, initial_cost, optimality,
nfev, njev, status].  The scene is generated from --seed, so the same arguments give the same inputs on every run.  With --gpus N > 1
frame_rt holds rank 0's frames.
The library must have been built by __graft_entry__.build(); the benchmark compiles nothing and writes nothing into the tree.
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

METRIC, UNIT = "reprojection_residuals_per_sec", "residuals/s"
BA_KW = dict(tolerance=1e-4, max_iterations=100, loss="linear", f_scale=1.0)
REF_FRAMES = {"cfg1": 20, "cfg2": 20, "cfg3": 12, "cfg4": 8, "cfg5": 2}      # CPU sample: ~10-40 s of scipy TRF + finite differences


def subsample_frames(scene, frames):
  s = dict(scene)
  s["F"] = len(frames)
  s["points"] = scene["points"][:, frames]; s["valid"] = scene["valid"][:, frames]
  s["frame_valid"] = scene["frame_valid"][frames]
  for k in ("init", "gt"):
    d = dict(scene[k]); d["frame_poses"] = scene[k]["frame_poses"][frames]; s[k] = d
  return s


def cpu_reference_step(scene):
  """One bundle_adjust of the reference's CPU path (its numpy + scipy restatement) on the host cores:
  (residuals/s, seconds, nfev, njev, corners)."""
  from oracle.ba_oracle import Problem
  prob = Problem.from_scene(scene, optimize=dict(cameras=True))
  t = time.perf_counter()
  _, res = prob.bundle_adjust(tolerance=BA_KW["tolerance"], max_iterations=BA_KW["max_iterations"], loss=BA_KW["loss"])
  dt = time.perf_counter() - t
  n = int(prob.inliers.sum())
  return n * (res.nfev + res.njev) / dt, dt, int(res.nfev), int(res.njev), n


def cpu_baseline_block(scene, workload, frames):
  """The CPU baseline on the first `frames` frames of the workload, after a small warm-up call (imports, caches)."""
  nf = min(scene["F"], frames)
  cpu_reference_step(subsample_frames(scene, np.arange(min(2, nf))))
  v, dt, nfev, njev, n = cpu_reference_step(subsample_frames(scene, np.arange(nf)))
  what = "oracle/ba_oracle.py: numpy restatement of evaluate + the identical scipy.optimize.least_squares call"
  return dict(value=v, unit=UNIT, cores=os.cpu_count(), kind="port",
              sample=f"{workload}: first {nf} of {scene['F']} frames ({n} corners), one full bundle_adjust ({nfev} nfev, {njev} njev, {dt:.1f} s); "
                     f"{what}; all {os.cpu_count()} host cores available to numpy / scipy / OpenCV's default thread pools, the Python-level algorithm is serial"), dt, nfev, njev, n


class ClockSampler(threading.Thread):
  """SM clock and throttle reasons sampled DURING the timed regions: NVML (1 ms period) when importable, else nvidia-smi."""
  REASONS = {0x4: "sw_power_cap", 0x8: "hw_slowdown", 0x20: "sw_thermal_slowdown", 0x40: "hw_thermal_slowdown"}

  def __init__(self, index=0):
    super().__init__(daemon=True)
    self.index, self.samples, self.reasons, self.stop_flag, self.max_mhz, self.source = index, [], set(), False, None, None

  def _run_nvml(self):
    import pynvml
    pynvml.nvmlInit()
    h = pynvml.nvmlDeviceGetHandleByIndex(self.index)
    self.max_mhz = float(pynvml.nvmlDeviceGetMaxClockInfo(h, pynvml.NVML_CLOCK_SM))
    get_reasons = getattr(pynvml, "nvmlDeviceGetCurrentClocksEventReasons", None) or pynvml.nvmlDeviceGetCurrentClocksThrottleReasons
    self.source = "nvml"
    while not self.stop_flag:
      self.samples.append(float(pynvml.nvmlDeviceGetClockInfo(h, pynvml.NVML_CLOCK_SM)))
      mask = int(get_reasons(h))
      for bit, name in self.REASONS.items():
        if mask & bit: self.reasons.add(name)
      time.sleep(0.001)

  def _run_smi(self):
    q = ("clocks.sm,clocks.max.sm,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
         "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")
    names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
    self.source = "nvidia-smi"
    while not self.stop_flag:
      try:
        out = subprocess.run(["nvidia-smi", f"--id={self.index}", f"--query-gpu={q}", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=5).stdout.strip().split(",")
        self.samples.append(float(out[0])); self.max_mhz = float(out[1])
        for n, v in zip(names, out[2:]):
          if "Active" in v and "Not" not in v: self.reasons.add(n)
      except Exception:
        pass
      time.sleep(0.05)

  def run(self):
    try:
      self._run_nvml()
    except Exception:
      if not self.stop_flag: self._run_smi()

  def summary(self):
    return dict(sm_mhz=float(np.median(self.samples)) if self.samples else None, sm_max_mhz=self.max_mhz,
                reasons=sorted(self.reasons), samples=len(self.samples), source=self.source)


HBM_PEAK_GBS = 3350.0      # H100 SXM data sheet: 3.35 TB/s of HBM3 (a peak, not a reached figure)


def run_reference(args):
  from multical_b200 import synthetic
  rank = int(os.environ.get("RANK", "0"))
  if rank != 0:
    return
  scene = synthetic.make_workload(args.workload, seed=args.seed)
  frames = args.ref_frames or REF_FRAMES.get(args.workload, 4)
  nf = min(scene["F"], frames)
  sample = subsample_frames(scene, np.arange(nf))
  for _ in range(max(1, min(args.warmup, 2))):
    cpu_reference_step(subsample_frames(scene, np.arange(min(2, nf))))
  tot_res, tot_t, nfev, njev = 0.0, 0.0, 0, 0
  t_start = time.perf_counter()
  steps_done = 0
  for _ in range(args.steps):
    v, dt, nf_, nj_, n = cpu_reference_step(sample)
    tot_res += n * (nf_ + nj_); tot_t += dt; nfev += nf_; njev += nj_; steps_done += 1
    if time.perf_counter() - t_start > args.ref_budget_s: break          # bounded: the whole run ends within minutes
  value = tot_res / tot_t
  what = "oracle/ba_oracle.py (numpy + the identical scipy call)"
  line = dict(metric=METRIC, value=value, unit=UNIT, n_gpus=args.gpus, steps=steps_done, warmup=args.warmup,
              ms_per_step=1e3 * tot_t / steps_done, higher_is_better=True, scaling="strong", vs_baseline=None, dtype="f64",
              data="synthetic", impl="reference",
              config=dict(workload=args.workload, sample=f"first {nf} of {scene['F']} frames, full bundle_adjust per step", corners=n,
                          steps_requested=args.steps, steps_run=steps_done, budget_s=args.ref_budget_s),
              lm_iters_per_sec=njev / tot_t,
              cpu_baseline=dict(value=value, unit=UNIT, cores=os.cpu_count(), kind="port",
                                sample=f"{args.workload}: first {nf} of {scene['F']} frames ({n} corners), {what}: scipy TRF + LSMR with 2-point "
                                       f"finite-difference Jacobian; all {os.cpu_count()} host cores available to the default thread pools of numpy / "
                                       f"scipy / OpenCV, the Python-level algorithm is serial"),
              e2e=dict(value=value, unit=UNIT, h2d_bytes_per_step=0, d2h_bytes_per_step=0))
  emit(line)


def run_ours(args):
  import torch
  import torch.distributed as dist
  from multical_b200 import synthetic
  from multical_b200.calibration import from_scene, get_engine
  from multical_b200.engine import Engine
  from multical_b200 import distributed as mdist

  rank = int(os.environ.get("RANK", "0")); world = int(os.environ.get("WORLD_SIZE", "1")); local = int(os.environ.get("LOCAL_RANK", "0"))
  assert world == args.gpus, f"--gpus {args.gpus} but WORLD_SIZE={world}"
  torch.cuda.set_device(local)
  os.environ["MCBA_DEVICE"] = str(local)
  if world > 1:
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
  stream = torch.cuda.current_stream()
  flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")      # > the 50 MB L2 of an H100
  NO_PREPARE = 256

  def barrier():
    if world > 1: dist.barrier()
    torch.cuda.synchronize()

  def allmax(x):
    tt = torch.tensor([x], dtype=torch.float64, device="cuda")
    if world > 1: dist.all_reduce(tt, op=dist.ReduceOp.MAX)
    return float(tt.item())

  def allsum_int(x):
    tt = torch.tensor([x], dtype=torch.int64, device="cuda")
    if world > 1: dist.all_reduce(tt)
    return int(tt.item())

  def pin(scene):
    # the step's inputs live in pinned host memory (the e2e timed region copies them to the device every step)
    for key in ("points", "valid"):
      scene[key] = torch.from_numpy(np.ascontiguousarray(scene[key])).pin_memory().numpy()
    return scene

  eng = get_engine(local)
  eng.lib.mcba_set_stream(eng.h, stream.cuda_stream)
  if world > 1:
    mdist.init_comm(eng, rank, world)

  def measure(local_scene, steps, warmup, e2e=True, roofline=True, dump_dir=None):
    """Device-resident solves, end-to-end solves and the linearisation kernel's roofline point for one (sharded) scene."""
    calib = from_scene(local_scene).enable(cameras=True)
    n_total = allsum_int(int(calib.inliers.sum()))
    state0 = calib._state_arrays()
    calib._upload(calib.inliers)

    def solve_resident():
      eng.set_params(*state0)
      flush.zero_()
      e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
      e0.record(stream)
      res = eng.solve(ftol=BA_KW["tolerance"], max_nfev=BA_KW["max_iterations"], loss=BA_KW["loss"], f_scale=BA_KW["f_scale"])
      e1.record(stream); e1.synchronize()
      return res, e0.elapsed_time(e1)
    for _ in range(warmup): solve_resident()
    barrier()
    t_dev, evals, njev, launches, last = 0.0, 0, 0, 0, None
    for _ in range(steps):
      res, ms = solve_resident()
      t_dev += ms; evals += res.nfev + res.njev; njev += res.njev; launches += res.kernel_launches; last = res
    if dump_dir and rank == 0:
      os.makedirs(dump_dir, exist_ok=True)
      for name, a in zip(("cam_rt", "board_rt", "frame_rt", "intrinsics"), eng.get_params()):
        np.save(os.path.join(dump_dir, name + ".npy"), np.asarray(a, dtype=np.float64))
      np.save(os.path.join(dump_dir, "solve.npy"),
              np.array([last.cost, last.initial_cost, last.optimality, last.nfev, last.njev, last.status], dtype=np.float64))
    barrier()
    t_dev = allmax(t_dev)
    out = dict(corners=n_total, ms_per_step=t_dev / steps, value=n_total * evals / (t_dev * 1e-3), lm_iters_per_sec=njev / (t_dev * 1e-3),
               nfev_plus_njev_per_step=evals / steps, gpu_launches=launches, cost=last.cost, nfev=last.nfev, params=eng.num_params)
    if e2e:
      def solve_e2e():
        c = from_scene(local_scene).enable(cameras=True)      # fresh object: nothing cached on host or device
        t0 = time.perf_counter()
        o = c.bundle_adjust(**BA_KW)          # returns after the device->host read of the solved parameters
        _ = o.last_solve.cost
        torch.cuda.synchronize()
        return o.last_solve, time.perf_counter() - t0
      for _ in range(warmup): solve_e2e()
      barrier()
      t_e2e, evals_e, njev_e = 0.0, 0, 0
      for _ in range(steps):
        flush.zero_(); torch.cuda.synchronize()
        res, dt = solve_e2e(); t_e2e += dt; evals_e += res.nfev + res.njev; njev_e += res.njev
      barrier()
      t_e2e = allmax(t_e2e)
      # dense upload: mask (1 B/entry) + observations (16 B/entry) of the [C,F,B,P] table, board points, parameter state
      h2d = int(calib.inliers.size) * (1 + 16) + int(np.prod(calib.board_points.points.shape)) * 8 + sum(a.size for a in state0) * 8
      out["e2e"] = dict(value=n_total * evals_e / t_e2e, unit=UNIT, h2d_bytes_per_step=h2d, d2h_bytes_per_step=eng.num_params * 8 + 64,
                        ms_per_step=1e3 * t_e2e / steps, lm_iters_per_sec=njev_e / t_e2e)
    if roofline:
      calib._upload(calib.inliers)
      info = eng.bench_info(0)
      eng.bench_launch(0, 3)                      # builds the pose tables, warms up
      times = []
      for _ in range(10):
        flush.zero_()                             # evict the inputs between timed launches
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream); eng.bench_launch(0 | NO_PREPARE, 1); e1.record(stream); e1.synchronize()
        times.append(e0.elapsed_time(e1) * 1e-3)
      dur = float(np.mean(times))
      ach = info["bytes_per_launch"] / dur / 1e9
      out["roofline"] = dict(bound="hbm", achieved=ach, peak=HBM_PEAK_GBS, unit="GB/s", frac=ach / HBM_PEAK_GBS, bytes_per_launch=info["bytes_per_launch"],
                             launch_ms=dur * 1e3, launches_per_step=out["nfev_plus_njev_per_step"] / 2.0)
    return out, calib

  sampler = ClockSampler(local); sampler.start()
  # ---- main workload: the same scene at every N, frames sharded over the ranks ----------------------------------------------
  scene = synthetic.make_workload(args.workload, seed=args.seed)
  my = mdist.frame_range(scene["F"], rank, world)
  local_scene = pin(subsample_frames(scene, np.arange(*my)) if world > 1 else scene)
  main, calib = measure(local_scene, args.steps, args.warmup, dump_dir=args.dump_outputs)

  # the same end-to-end call over a float32 table: make_point_table keeps the dtype of the detector's corners (tables.py:15-17; cv2 returns
  # float32), so for real detections THIS is the reference's table.  The scene is the main scene rounded to float32 (8 B per entry over the link).
  e2e_f32 = None
  if args.secondary:
    scene32 = dict(local_scene)
    scene32["points"] = torch.from_numpy(np.ascontiguousarray(local_scene["points"], dtype=np.float32)).pin_memory().numpy()
    def solve_e2e32():
      c = from_scene(scene32).enable(cameras=True)
      t0 = time.perf_counter()
      o = c.bundle_adjust(**BA_KW)
      _ = o.last_solve.cost
      torch.cuda.synchronize()
      return o.last_solve, time.perf_counter() - t0
    for _ in range(args.warmup): solve_e2e32()
    barrier()
    t32, ev32 = 0.0, 0
    for _ in range(args.steps):
      flush.zero_(); torch.cuda.synchronize()
      r32, dt = solve_e2e32(); t32 += dt; ev32 += r32.nfev + r32.njev
    barrier()
    t32 = allmax(t32)
    e2e_f32 = dict(value=main["corners"] * ev32 / t32, unit=UNIT, ms_per_step=1e3 * t32 / args.steps,
                   h2d_bytes_per_step=int(calib.inliers.size) * (1 + 8) + int(np.prod(calib.board_points.points.shape)) * 8 + sum(a.size for a in calib._state_arrays()) * 8,
                   note="point table as float32 (the dtype the reference's make_point_table keeps for cv2 detections); `e2e` above is the float64 table")

  others = {}
  parity = None
  if world == 1 and args.secondary:
    for wl in ("cfg2", "cfg3", "cfg5"):      # cfg5 = BASELINE configs[4] (64 cameras x 2000 frames, 50.8 M corners, n_s = 1030): it fits one GPU as well
      if wl == args.workload: continue
      o, _ = measure(pin(synthetic.make_workload(wl, seed=args.seed)), args.steps, args.warmup)
      o.pop("cost", None)
      others[wl] = o
  if world > 1:
    # the sharded solve must be the single-GPU solve: rank 0 solves the whole scene alone on a second context
    if rank == 0:
      from multical_b200 import calibration as _cal
      solo = Engine(local, stream=stream.cuda_stream)            # second context on this GPU: no communicator, the whole scene
      saved = _cal._engines.get(local)
      _cal._engines[local] = solo
      try:
        ref_res = from_scene(scene).enable(cameras=True).bundle_adjust(**BA_KW).last_solve
      finally:
        _cal._engines[local] = saved
        solo.close()
      rel = abs(main["cost"] - ref_res.cost) / ref_res.cost
      parity = dict(single_gpu_cost=ref_res.cost, sharded_cost=main["cost"], rel_diff=rel, single_gpu_nfev=ref_res.nfev, sharded_nfev=main["nfev"])
      assert rel <= 1e-9 and ref_res.nfev == main["nfev"], f"the {world}-rank solve differs from the single-GPU solve: {parity}"
    barrier()
    if args.secondary:
      # weak scaling: cfg2's 200 frames per GPU, cameras / boards (shared parameters) common
      base = dict(synthetic.WORKLOADS["cfg2"])
      wscene = synthetic.make_scene(seed=args.seed, **{**base, "F": base["F"] * world})
      wmy = mdist.frame_range(wscene["F"], rank, world)
      o, _ = measure(pin(subsample_frames(wscene, np.arange(*wmy))), args.steps, args.warmup, e2e=False, roofline=False)
      o.pop("cost", None)
      others["weak_cfg2_per_gpu"] = dict(o, scaling="weak", frames_per_gpu=base["F"])
  sampler.stop_flag = True; sampler.join(timeout=2)

  if rank != 0:
    if world > 1: dist.destroy_process_group()
    return

  roofline = dict(main["roofline"], peak_source="H100 SXM data sheet (3.35 TB/s HBM3)",
                  kernel="k_linearize (fused: residuals + analytic Jacobian + per-view moment SYRK on the fp64 tensor path + twist-map expansion into "
                         "H_ff / W / shared records; reads every corner once, writes nothing per corner or per view)",
                  algorithmic_bytes="18 B/corner (16 B observation f64x2 + 2 B point index) + 16 B/view, one launch per evaluation",
                  note="the bound named is HBM; the pass needs ~160 DFMA + 12 DMMA(m8n8k4) per corner against 18 B (~60 flop/B vs an fp64 ridge of "
                       "~10 flop/B on an H100 SXM: 34 TFLOP/s fp64 over 3.35 TB/s, data sheet), so the fp64 pipe bounds it")

  # ---- CPU baseline: the reference's path on a bounded sample of the same workload ---------------------------------------------
  cpu_baseline, *_ = cpu_baseline_block(scene, args.workload, args.ref_frames or REF_FRAMES.get(args.workload, 4))

  line = dict(metric=METRIC, value=main["value"], unit=UNIT, n_gpus=world, steps=args.steps, warmup=args.warmup,
              ms_per_step=main["ms_per_step"], higher_is_better=True, scaling="strong", vs_baseline=None, dtype="f64",
              data="synthetic",
              config=dict(workload=args.workload, cameras=scene["C"], frames=scene["F"], boards=scene["B"], corners=main["corners"],
                          params=main["params"] if world == 1 else None, frames_per_gpu=my[1] - my[0], camera_model=scene["model"],
                          solver="TRF semantics (ftol=1e-4, x_scale=jac, max_nfev=100), exact Schur inner solve; device-resident loop (CUDA-graph WHILE)",
                          l2="flushed between timed iterations (256 MiB write)", seed=args.seed,
                          parallelism=f"frames sharded over {world} GPU(s); in-kernel NVLink peer-memory exchanges" if world > 1 else "1 GPU"),
              lm_iters_per_sec=main["lm_iters_per_sec"], nfev_plus_njev_per_step=main["nfev_plus_njev_per_step"],
              e2e=main["e2e"], gpu_launches=main["gpu_launches"], clocks=sampler.summary(), roofline=roofline, cpu_baseline=cpu_baseline)
  if e2e_f32: line["e2e_float32_table"] = e2e_f32
  if others: line["other_workloads"] = others
  if parity: line["parity_vs_single_gpu"] = parity
  emit(line)
  if world > 1: dist.destroy_process_group()


_REAL_STDOUT = None


def emit(line):
  """The one JSON line goes to the real stdout; everything else this process (or NCCL) prints was sent to stderr."""
  out = os.fdopen(os.dup(_REAL_STDOUT), "w") if _REAL_STDOUT is not None else sys.stdout
  out.write(json.dumps(line) + "\n"); out.flush()


def main():
  global _REAL_STDOUT
  # libraries (NCCL's version banner, torchrun warnings) may write to fd 1: keep stdout clean for the single JSON line
  sys.stdout.flush()
  _REAL_STDOUT = os.dup(1)
  os.dup2(2, 1)
  ap = argparse.ArgumentParser()
  ap.add_argument("--gpus", type=int, default=1)
  ap.add_argument("--steps", type=int, default=10)
  ap.add_argument("--warmup", type=int, default=3)
  ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
  ap.add_argument("--workload", default="cfg4")
  ap.add_argument("--seed", type=int, default=0)
  ap.add_argument("--ref-frames", type=int, default=0, help="frames in the CPU-baseline sample (0: per-workload default)")
  ap.add_argument("--ref-budget-s", type=float, default=240.0, help="the reference arm stops taking steps after this many seconds")
  ap.add_argument("--no-secondary", dest="secondary", action="store_false", help="skip the secondary workload blocks")
  ap.add_argument("--dump-outputs", default=None, metavar="DIR", help="write the main workload's last timed solve as DIR/<name>.npy")
  args = ap.parse_args()
  if args.impl == "reference":
    run_reference(args)
  else:
    run_ours(args)


if __name__ == "__main__":
  main()
