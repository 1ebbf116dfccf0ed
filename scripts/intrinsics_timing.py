"""Time the single-camera intrinsic calibration (multical_b200/intrinsics.py) on the GPU against cv2.calibrateCameraExtended on the host.

  python scripts/intrinsics_timing.py [--out DIR]

Per case (synthetic scenes, 0.3 px noise):
  round        one round of the loop for every camera at once: intrinsic_init (one launch chain for all cameras) + one solve and the
               view errors per camera.  init_ms = host clock around mcba_intrinsic_init (ends in a stream synchronise), solve_ms = the
               engine's CUDA-event time of each solve, round_ms = host clock around the whole round (uploads included).
  end_to_end   host clock around calibrate_cameras(..., intrinsic_error_limit=1.0) from the nested detections, host work included (one
               round: the RMS of these scenes is below 1 px).
  opencv       cv2.calibrateCameraExtended with the reference's criteria (EPS + MAX_ITER, 10, 1e-3), one camera, on this host's CPU.
The GPU's name, power limit and SM clock are printed with the numbers."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from multical_b200 import intrinsics, synthetic  # noqa: E402
from multical_b200.board import Board  # noqa: E402
from multical_b200.structs import struct  # noqa: E402


def detections(scene, c):
  pts, valid = scene["points"][c].astype(np.float32), scene["valid"][c]
  return [[struct(corners=pts[f, b][valid[f, b]], ids=np.flatnonzero(valid[f, b])) for b in range(scene["B"])] for f in range(scene["F"])]


def gpu_info():
  q = "name,power.limit,clocks.max.sm,clocks.sm"
  try:
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout
    return out.strip().splitlines()[0]
  except Exception as e:       # the timing itself still needs the GPU; only the label is missing
    return f"unavailable ({e})"


def time_case(name, scene, boards, repeats=3):
  C = scene["C"]
  dets = [detections(scene, c) for c in range(C)]
  views = [intrinsics.calibration_points(boards, dets[c]) for c in range(C)]
  sizes = [scene["image_size"]] * C
  eng = intrinsics.intrinsics_engine()
  real_init = eng.intrinsic_init
  init_ms = []
  def timed_init(*a, **k):
    t = time.perf_counter(); out = real_init(*a, **k); init_ms.append(1e3 * (time.perf_counter() - t)); return out
  eng.intrinsic_init = timed_init
  intrinsics.calibrate_views(boards, views, sizes)          # warm-up: module load, buffer allocation
  rounds = []
  for _ in range(repeats):
    init_ms.clear()
    t = time.perf_counter()
    res = intrinsics.calibrate_views(boards, views, sizes)
    rounds.append(dict(round_ms=1e3 * (time.perf_counter() - t), init_ms=init_ms[0], solve_ms=[r.solve.device_ms for r in res],
                       nfev=[r.solve.nfev for r in res]))
  eng.intrinsic_init = real_init
  e2e = []
  for _ in range(repeats):
    t = time.perf_counter()
    intrinsics.calibrate_cameras(boards, dets, sizes, 1.0)
    e2e.append(1e3 * (time.perf_counter() - t))
  return dict(case=name, cameras=C, views_per_camera=[len(v) for v in views], corners_per_camera=[int(sum(x.ids.size for x in v)) for v in views],
              rounds=rounds, end_to_end_ms=e2e, rms=[float(r.rms) for r in res])


def time_opencv(scene, boards, n_views):
  import cv2
  views = intrinsics.calibration_points(boards, detections(scene, 0))[:n_views]
  op = [v.object_points.reshape(-1, 1, 3) for v in views]
  ip = [v.corners.reshape(-1, 1, 2) for v in views]
  t = time.perf_counter()
  rms = cv2.calibrateCameraExtended(op, ip, tuple(scene["image_size"]), None, None,
                                    criteria=(cv2.TERM_CRITERIA_EPS + cv2.TERM_CRITERIA_MAX_ITER, 10, 1e-3), flags=0)[0]
  return dict(case=f"opencv_{len(views)}_views", views=len(views), corners=int(sum(v.ids.size for v in views)),
              seconds=time.perf_counter() - t, rms=float(rms), cv2=cv2.__version__)


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--out", default=None)
  args = ap.parse_args()
  results = [dict(gpu=gpu_info())]
  cfg2 = synthetic.make_workload("cfg2")                                    # 4 cameras x 200 frames, one ChArUco board
  b2 = [Board(p, size=(16, 22)) for p in cfg2["board_points"]]
  results.append(time_case("cfg2_sized", cfg2, b2))
  cfg4 = synthetic.make_scene(C=2, F=1000, boards=("cube", 10, 10, 0.04, 5), rig="dome", vis=0.85, seed=0)   # cfg4's rig, 2 of its cameras
  b4 = [Board(p, size=(9, 9)) for p in cfg4["board_points"]]
  results.append(time_case("cfg4_sized", cfg4, b4))
  for n in (50, 200):
    results.append(time_opencv(cfg2, b2, n))
  results.append(dict(gpu_after=gpu_info()))
  for r in results: print(json.dumps(r))
  if args.out:
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "intrinsics_timing.json"), "w") as fh:
      json.dump(results, fh, indent=1)


if __name__ == "__main__":
  main()
