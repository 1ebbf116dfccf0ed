"""Time stereo_calibrate (multical_b200/stereo.py) on the GPU against cv2.stereoCalibrate with the reference's criteria (60, 1e-6) and
flags (fixed intrinsics) on the same host, for a 2-camera synthetic pair (synthetic.make_scene(C=2, vis=0.4)) at each view count.

  python scripts/stereo_timing.py [--views 200 1000] [--repeats 3]

  start        host clock around mcba_stereo_init (per-view PnP of both cameras and the median relative pose; copies included)
  solve        device time of the engine's solve (CUDA events, SolveInfo.device_ms)
  end_to_end   host clock around stereo_calibrate, from the per-view lists to the returned cameras and pose
  opencv       host clock around cv2.stereoCalibrate on this host's CPU
The median over the repeats is printed, after one warm-up call, with the RMS of both and the GPU's name, power limit and SM clocks."""
import argparse
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from intrinsics_timing import gpu_info  # noqa: E402
from multical_b200 import stereo, synthetic  # noqa: E402
from multical_b200.camera import stereo_calibrate  # noqa: E402
from test_gpu_stereo import cameras_of, cv_stereo, matches_of  # noqa: E402


def time_pair(F, repeats):
  scene = synthetic.make_scene(C=2, F=F, vis=0.4, seed=5)
  m = matches_of(scene)
  cams = cameras_of(scene)
  intr = np.stack([stereo._camera_params(c, "standard") for c in cams])
  problem = stereo.pair_problem(m)
  stereo_calibrate(cams, m)
  start, solve, e2e, cv = [], [], [], []
  for _ in range(repeats):
    t0 = time.perf_counter(); stereo.stereo_init("standard", intr, problem); start.append(time.perf_counter() - t0)
    solve.append(stereo.solve_pair("standard", intr, problem).solve.device_ms * 1e-3)
    t0 = time.perf_counter(); _, _, _, err = stereo_calibrate(cams, m); e2e.append(time.perf_counter() - t0)
  for _ in range(max(1, repeats // 3)):
    t0 = time.perf_counter(); err_cv = cv_stereo(cams, m, (3, 60, 1e-6))[0]; cv.append(time.perf_counter() - t0)
  ms = lambda v: f"{np.median(v) * 1e3:.2f} ms"
  n = sum(len(o) for o in m.object_points)
  print(f"2 x {len(m.object_points)} views ({n} corners per camera): start {ms(start)}, solve {ms(solve)} (device), end to end {ms(e2e)}; "
        f"cv2.stereoCalibrate {ms(cv)}; RMS device {err:.6f}, OpenCV {err_cv:.6f}")


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--views", type=int, nargs="+", default=[200, 1000])
  ap.add_argument("--repeats", type=int, default=3)
  a = ap.parse_args()
  print("GPU:", gpu_info())
  for F in a.views: time_pair(F, a.repeats)


if __name__ == "__main__":
  main()
