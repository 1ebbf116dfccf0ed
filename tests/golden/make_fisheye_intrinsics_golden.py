"""Generate the golden vectors of the fisheye intrinsic calibration (tests/test_gpu_fisheye_intrinsics.py) from the UNMODIFIED reference
`CameraFisheye.calibrate` (multical/camera_fisheye.py:70-94), imported through tests/refshim.

Run with MULTICAL_REFERENCE pointing at a checkout of multical:
    MULTICAL_REFERENCE=<path> python tests/golden/make_fisheye_intrinsics_golden.py
Each case stores the detections of one camera (a synthetic fisheye scene), the call's arguments and what the reference returns:
  K, dist, err, and the views it handed to cv2.fisheye.calibrate (view_sizes: corners per view in order; view_corners, view_object_points:
  all of them concatenated), recorded by wrapping cv2.fisheye.calibrate for the call.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "refshim"))

from multical_b200 import synthetic  # noqa: E402
from multical_b200.board import Board  # noqa: E402
import loader  # noqa: E402

CUBE = dict(boards=("cube", 10, 10, 0.04, 5), rig="dome")
CASES = {
  # name: scene, board size and min_points, calibrate() keyword arguments, numpy seed for max_images.  model / fix_aspect are stored on
  # the camera and never reach OpenCV: fisheye_small_12 sets both to show it.
  "fisheye_small_12": dict(scene=dict(C=1, F=12, vis=0.85, seed=81, model="fisheye"), board=((16, 22), 20),
                           kw=dict(model="fix_k2", fix_aspect=True)),
  "fisheye_40": dict(scene=dict(C=1, F=40, vis=0.85, seed=82, model="fisheye"), board=((16, 22), 20), kw=dict()),
  "fisheye_max_images_36": dict(scene=dict(C=1, F=36, vis=0.85, seed=83, model="fisheye"), board=((16, 22), 20),
                                kw=dict(max_images=20), np_seed=11),
  "fisheye_cube_10": dict(scene=dict(C=1, F=10, vis=0.8, seed=84, model="fisheye", **CUBE), board=((9, 9), 12), kw=dict()),
}


def make_case(ref, name, spec):
  scene = synthetic.make_scene(**spec["scene"])
  pts, valid = scene["points"][0], scene["valid"][0]
  size, min_points = spec["board"]
  boards = [Board(p, size=size, min_points=min_points) for p in scene["board_points"]]
  pts = np.where(valid[..., None], pts, 0.0).astype(np.float32)
  dets = [[ref.struct(corners=pts[f, b][valid[f, b]], ids=np.flatnonzero(valid[f, b])) for b in range(scene["B"])] for f in range(scene["F"])]
  import multical.camera_fisheye as reffish
  calls = []
  real = reffish.cv2.fisheye.calibrate
  def recorded(objpoints, corners, *a, **k):
    calls.append((objpoints, corners))
    return real(objpoints, corners, *a, **k)
  reffish.cv2.fisheye.calibrate = recorded
  try:
    if "np_seed" in spec: np.random.seed(spec["np_seed"])
    cam, err = ref.CameraFisheye.calibrate(boards, dets, tuple(scene["image_size"]), **spec["kw"])
  finally:
    reffish.cv2.fisheye.calibrate = real
  assert len(calls) == 1
  op, ip = calls[0]
  kw = spec["kw"]
  out = dict(points=pts, valid=valid, board_points=np.stack(scene["board_points"]), board_size=np.array(size), min_points=min_points,
             image_size=np.array(scene["image_size"]), model=kw.get("model", "standard"), fix_aspect=kw.get("fix_aspect", False),
             max_images=kw.get("max_images", -1), np_seed=spec.get("np_seed", -1),
             K=np.asarray(cam.intrinsic), dist=np.asarray(cam.dist), err=float(err), cam_model=cam.model, cam_fix_aspect=cam.fix_aspect,
             view_sizes=np.array([c.shape[1] for c in ip]), view_corners=np.concatenate([c[0] for c in ip]),
             view_object_points=np.concatenate([o[0] for o in op]), gt_K=scene["gt"]["K"][0], gt_dist=scene["gt"]["dist"][0])
  np.savez_compressed(os.path.join(HERE, f"{name}.npz"), **out)
  print(name, "views", len(ip), "err", err, "K", np.asarray(cam.intrinsic)[[0, 1, 0, 1], [0, 1, 2, 2]], "dist", np.ravel(cam.dist))


def main(names):
  ref = loader.load()
  # calibration_points (camera.py:229-235) joins the boards' views with `+` on structs, which py-structs defines key by key
  # (Struct._zipWith(operator.add)); the shared shim's Struct has no `+`, so it is added here, in this process only
  import operator
  from structs.struct import Struct
  Struct.__add__ = lambda a, b: a._zipWith(operator.add, b)
  for n in names or CASES:
    make_case(ref, n, CASES[n])


if __name__ == "__main__":
  main(sys.argv[1:])
