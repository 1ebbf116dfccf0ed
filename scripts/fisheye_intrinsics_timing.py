"""Time the fisheye intrinsic calibration (multical_b200/intrinsics.py calibrate_cameras_fisheye) on the GPU against cv2.fisheye.calibrate
on the host, at cfg3's size (8 fisheye cameras x 500 frames, one ChArUco board, 0.3 px noise).

  python scripts/fisheye_intrinsics_timing.py [--out DIR] [--cameras C] [--frames F]

  round        calibrate_views for every camera at once: mcba_intrinsic_init (one launch chain for all cameras) + one solve and the view
               errors per camera.  init_ms = host clock around mcba_intrinsic_init (ends in a stream synchronise), solve_ms = the engine's
               CUDA-event time of each solve, round_ms = host clock around the whole call (uploads included).
  end_to_end   host clock around calibrate_cameras_fisheye from the nested detections, host work included.
  opencv       cv2.fisheye.calibrate with the reference's criteria (EPS + MAX_ITER, 10, 1e-3) and flags, for each of the first two
               cameras' views, on this host's CPU.
The GPU's name, power limit and SM clocks are printed with the numbers."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from intrinsics_timing import detections, gpu_info  # noqa: E402
from multical_b200 import intrinsics, synthetic  # noqa: E402
from multical_b200.board import Board  # noqa: E402


def time_round(scene, boards, repeats=3):
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
  intrinsics.calibrate_views(boards, views, sizes, model="fisheye")          # warm-up: module load, buffer allocation
  rounds = []
  for _ in range(repeats):
    init_ms.clear()
    t = time.perf_counter()
    res = intrinsics.calibrate_views(boards, views, sizes, model="fisheye")
    rounds.append(dict(round_ms=1e3 * (time.perf_counter() - t), init_ms=init_ms[0], solve_ms=[r.solve.device_ms for r in res],
                       nfev=[r.solve.nfev for r in res]))
  eng.intrinsic_init = real_init
  e2e = []
  for _ in range(repeats):
    t = time.perf_counter()
    _, errs = intrinsics.calibrate_cameras_fisheye(boards, dets, sizes)
    e2e.append(1e3 * (time.perf_counter() - t))
  return dict(case=f"cfg3_sized_{C}x{scene['F']}", cameras=C, views_per_camera=[len(v) for v in views],
              corners_per_camera=[int(sum(x.ids.size for x in v)) for v in views], rounds=rounds, end_to_end_ms=e2e, rms=[float(e) for e in errs])


def time_opencv(scene, boards, c):
  import cv2
  views = intrinsics.calibration_points(boards, detections(scene, c))
  flags = cv2.fisheye.CALIB_RECOMPUTE_EXTRINSIC | cv2.fisheye.CALIB_FIX_SKEW
  t = time.perf_counter()
  try:
    rms = float(cv2.fisheye.calibrate([v.object_points[None] for v in views], [v.corners[None] for v in views], tuple(scene["image_size"]),
                                      None, None, criteria=(cv2.TERM_CRITERIA_EPS + cv2.TERM_CRITERIA_MAX_ITER, 10, 1e-3), flags=flags)[0])
  except cv2.error as e:
    rms = f"raised: {str(e).strip().splitlines()[-1]}"
  return dict(case=f"opencv_camera_{c}", views=len(views), corners=int(sum(v.ids.size for v in views)), seconds=time.perf_counter() - t,
              rms=rms, cv2=cv2.__version__)


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--out", default=None)
  ap.add_argument("--cameras", type=int, default=8)
  ap.add_argument("--frames", type=int, default=500)
  args = ap.parse_args()
  results = [dict(gpu=gpu_info())]
  scene = synthetic.make_workload("cfg3", C=args.cameras, F=args.frames)
  boards = [Board(p, size=(16, 22), min_points=20) for p in scene["board_points"]]
  results.append(time_round(scene, boards))
  for c in range(min(2, args.cameras)):
    results.append(time_opencv(scene, boards, c))
  results.append(dict(gpu_after=gpu_info()))
  for r in results: print(json.dumps(r))
  if args.out:
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "fisheye_intrinsics_timing.json"), "w") as fh:
      json.dump(results, fh, indent=1)


if __name__ == "__main__":
  main()
