"""Launch the hot kernels a few times on one workload (target for a profiler; MCBA_PROF=1 prints k_lm phase stamps)."""
import os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from multical_b200 import synthetic
from multical_b200.calibration import from_scene

wl = sys.argv[1] if len(sys.argv) > 1 else "cfg2"
mode = sys.argv[2] if len(sys.argv) > 2 else "kernels"
t = time.time()
scene = synthetic.make_workload(wl)
calib = from_scene(scene).enable(cameras=True)
print(wl, "corners", int(scene["valid"].sum()), "gen %.1fs" % (time.time() - t), flush=True)
t = time.time()
eng = calib._upload(calib.inliers)
print("upload %.3fs" % (time.time() - t), flush=True)
if mode == "kernels":
  for _ in range(3):
    eng.bench_launch(0, 1)      # linearise: k_prepare + k_views<MOMENTS> parts
    eng.bench_launch(2, 1)      # trial cost: k_prepare + k_views<COST>
  eng.residuals()
elif mode == "time":            # CUDA-event time of the linearisation kernel alone (what bench.py reports as roofline.launch_ms)
  import torch
  stream = torch.cuda.Stream()
  eng.lib.mcba_set_stream(eng.h, stream.cuda_stream)
  flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
  eng.bench_launch(0, 3)
  ts = []
  with torch.cuda.stream(stream):
    for _ in range(10):
      flush.zero_()
      e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
      e0.record(stream); eng.bench_launch(0 | 256, 1); e1.record(stream); e1.synchronize()
      ts.append(e0.elapsed_time(e1) * 1e3)
  info = eng.bench_info(0)
  med = float(np.median(ts))
  print("moments=%s linearise kernel: median %.1f us (min %.1f) over %d corners -> %.1f GB/s algorithmic" % (
    os.environ.get("MCBA_MOMENTS", "mma"), med, min(ts), info["corners"], info["bytes_per_launch"] / med / 1e3), flush=True)
else:
  import torch
  for i in range(3):
    eng.set_params(*calib._state_arrays())
    t = time.time(); res = eng.solve(ftol=1e-4, max_nfev=100); dt = time.time() - t
    print("solve", i, "cost %.6f nfev %d njev %d status %d dev_ms %.3f wall_ms %.3f launches %d" % (res.cost, res.nfev, res.njev, res.status, res.device_ms, dt * 1e3, res.kernel_launches), flush=True)
