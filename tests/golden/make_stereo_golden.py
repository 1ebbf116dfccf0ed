"""Generate the golden vectors of stereo calibration (tests/test_gpu_stereo.py) from the UNMODIFIED reference `stereo_calibrate`
(multical/camera.py:261-286) called through `stereo_calibrate_detections` (multical/image/detect.py:45-59), imported through tests/refshim.

Run with MULTICAL_REFERENCE pointing at a checkout of multical:
    MULTICAL_REFERENCE=<path> python tests/golden/make_stereo_golden.py
Each case stores the detections of a synthetic two-camera scene with one board, the input cameras, the call's arguments and what the
reference returns (K, dist of both cameras, the 4x4 pose, err), and the frames stereo_calibrate_detections kept with their corner counts,
recorded by wrapping the stereo_calibrate it calls.
"""
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "refshim"))

from multical_b200 import synthetic  # noqa: E402
import loader  # noqa: E402

CASES = {
  # name: scene, stereo_calibrate keyword arguments, relative jitter of the input focal lengths (free intrinsics start off the truth),
  # frames the right camera does not see
  "stereo_standard_fixed": dict(scene=dict(C=2, F=30, vis=0.4, seed=61), kw=dict(), unseen=[3, 17]),
  "stereo_standard_free": dict(scene=dict(C=2, F=30, vis=0.5, seed=62), kw=dict(fix_intrinsic=False), jitter=0.01),
  "stereo_rational_fixed": dict(scene=dict(C=2, F=30, vis=0.4, seed=63, model="rational"), kw=dict()),
}


def make_case(ref, name, spec):
  scene = synthetic.make_scene(**spec["scene"])
  pts = np.where(scene["valid"][..., None], scene["points"], 0.0).astype(np.float32)[:, :, 0]      # [2, F, P, 2], one board
  valid = scene["valid"][:, :, 0].copy()
  valid[1, spec.get("unseen", [])] = False                      # frames the right camera misses: stereo_calibrate_detections drops them
  board_points = scene["board_points"][0].astype(np.float32)     # a ChArUco board's points are float32; OpenCV 4.13 refuses float64 ones
  dets = [[ref.struct(corners=pts[c, f][valid[c, f]], ids=np.flatnonzero(valid[c, f])) for f in range(scene["F"])] for c in range(2)]
  K, dist = scene["gt"]["K"].copy(), scene["gt"]["dist"].copy()
  rng = np.random.default_rng(1)
  if spec.get("jitter"):
    K[:, 0, 0] *= 1 + rng.normal(0, spec["jitter"], 2); K[:, 1, 1] = K[:, 0, 0]
  size, model = tuple(scene["image_size"]), scene["model"]
  # cv2.stereoCalibrate writes K and dist into the arrays it is given, which the reference's cameras hold: hand it copies
  cams = [ref.Camera(image_size=size, intrinsic=K[c].copy(), dist=dist[c].copy(), model=model) for c in range(2)]
  import multical.image.detect as detect
  calls = []
  real = detect.stereo_calibrate
  def recorded(cameras, matches, **kw):
    calls.append(matches)
    return real(cameras, matches, **kw)
  detect.stereo_calibrate = recorded
  try:
    left, right, pose, err = detect.stereo_calibrate_detections(dets, types.SimpleNamespace(points=board_points), cams, 0, 1, **spec["kw"])
  finally:
    detect.stereo_calibrate = real
  assert len(calls) == 1
  m = calls[0]
  kept = [f for f in range(scene["F"]) if np.intersect1d(dets[0][f].ids, dets[1][f].ids).size]
  assert [len(o) for o in m.object_points] == [np.intersect1d(dets[0][f].ids, dets[1][f].ids).size for f in kept]
  out = dict(points=pts, valid=valid, board_points=board_points, image_size=np.array(size), model=model, K_in=K, dist_in=dist,
             fix_intrinsic=spec["kw"].get("fix_intrinsic", True), fix_aspect=spec["kw"].get("fix_aspect", False),
             K1=np.asarray(left.intrinsic), d1=np.asarray(left.dist), K2=np.asarray(right.intrinsic), d2=np.asarray(right.dist),
             pose=np.asarray(pose), err=float(err), frames=np.array(kept), view_sizes=np.array([len(o) for o in m.object_points]))
  np.savez_compressed(os.path.join(HERE, f"{name}.npz"), **out)
  print(name, "views", len(kept), "err", err, "T", np.asarray(pose)[:3, 3])


def main(names):
  ref = loader.load()
  # multical/image/__init__.py imports the display helpers (matplotlib, Qt): skip it as the loader skips the package roots
  if "multical.image" not in sys.modules:
    p = types.ModuleType("multical.image")
    p.__path__ = [loader.REFERENCE_ROOT + "/multical/image"]
    sys.modules["multical.image"] = p
  for n in names or CASES:
    make_case(ref, n, CASES[n])


if __name__ == "__main__":
  main(sys.argv[1:])
