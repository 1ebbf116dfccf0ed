"""Generate the golden vectors of the single-camera intrinsic calibration (tests/test_gpu_intrinsics.py) from the UNMODIFIED reference
`Camera.calibrate` (multical/camera.py:68-105), imported through tests/refshim.

Run with MULTICAL_REFERENCE pointing at a checkout of multical:
    MULTICAL_REFERENCE=<path> python tests/golden/make_intrinsics_golden.py
Each case stores the detections of one camera (a synthetic scene; some views get several pixels of extra noise so that the 95 % view
cut of every round has a wide margin), the call's arguments and what the reference returns:
  K, dist, err, error_perview, board_ids, image_ids, rounds (calls of cv2.calibrateCameraExtended)
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

CASES = {
  # name: scene, {view frame: extra noise in px}, limit, calibrate() keyword arguments, numpy seed for max_images.  Every round of the
  # reference's loop drops exactly its two worst views; the extra noise makes those the noisy views of that round, each pair well apart
  # from the next, so that OpenCV's early stop cannot change which views a round drops.
  "intrinsics_loop_40": dict(scene=dict(C=1, F=40, vis=0.4, seed=65), outliers={3: 4.0, 17: 4.0, 29: 2.0, 8: 2.0, 33: 1.0, 12: 1.0},
                             limit=0.6, kw=dict(model="standard")),
  "intrinsics_small_12": dict(scene=dict(C=1, F=12, vis=0.4, seed=64), outliers={}, limit=0.2, kw=dict(model="standard")),
  "intrinsics_max_images_36": dict(scene=dict(C=1, F=36, vis=0.4, seed=63), outliers={}, limit=0.7,
                                   kw=dict(model="standard", max_images=24), np_seed=7, outliers_selected=(1.0, 1.0)),
}


def make_case(ref, name, spec):
  scene = synthetic.make_scene(**spec["scene"])
  pts, valid = scene["points"][0].copy(), scene["valid"][0]
  rng = np.random.default_rng(spec["scene"]["seed"] + 1000)
  boards = [Board(p, size=(16, 22)) for p in scene["board_points"]]
  outliers = dict(spec["outliers"])
  if "outliers_selected" in spec:         # noisy views among the ones max_images selects (the selection depends on coverage only)
    from multical_b200 import intrinsics
    from multical_b200.structs import struct
    np.random.seed(spec["np_seed"])
    views = intrinsics.calibration_points(boards, [[struct(corners=pts[f, b][valid[f, b]], ids=np.flatnonzero(valid[f, b]))
                                                    for b in range(scene["B"])] for f in range(scene["F"])])
    chosen = intrinsics.top_detection_coverage(views, spec["kw"]["max_images"], tuple(scene["image_size"]))
    outliers = {v.frame: s for v, s in zip(chosen[3::7], spec["outliers_selected"])}
  for f, sigma in outliers.items():
    pts[f] += rng.normal(0, sigma, pts[f].shape)
  pts = np.where(valid[..., None], pts, 0.0).astype(np.float32)
  dets = [[ref.struct(corners=pts[f, b][valid[f, b]], ids=np.flatnonzero(valid[f, b])) for b in range(scene["B"])] for f in range(scene["F"])]
  import multical.camera as refcam
  calls = []
  real = refcam.cv2.calibrateCameraExtended
  def counted(*a, **k):
    calls.append(1)
    return real(*a, **k)
  refcam.cv2.calibrateCameraExtended = counted
  try:
    if "np_seed" in spec: np.random.seed(spec["np_seed"])
    cam, err = ref.Camera.calibrate(boards, spec["limit"], dets, tuple(scene["image_size"]), **spec["kw"])
  finally:
    refcam.cv2.calibrateCameraExtended = real
  ds = cam.intrinsic_dataset
  assert not set(outliers) & set(ds["image_ids"]) and len(calls) == len(outliers) // 2 or not outliers, (name, len(calls), ds["image_ids"])
  out = dict(points=pts, valid=valid, board_points=np.stack(scene["board_points"]), image_size=np.array(scene["image_size"]),
             limit=spec["limit"], model=spec["kw"]["model"], max_images=spec["kw"].get("max_images", -1), np_seed=spec.get("np_seed", -1),
             K=np.asarray(cam.intrinsic), dist=np.asarray(cam.dist), err=float(err), error_perview=np.asarray(cam.error_perview).ravel(),
             board_ids=np.asarray(ds["board_ids"], np.float64), image_ids=np.asarray(ds["image_ids"], np.int64), rounds=len(calls))
  np.savez_compressed(os.path.join(HERE, f"{name}.npz"), **out)
  print(name, "rounds", len(calls), "err", err, "views", len(ds["image_ids"]))


def main(names):
  ref = loader.load()
  for n in names or CASES:
    make_case(ref, n, CASES[n])


if __name__ == "__main__":
  main(sys.argv[1:])
