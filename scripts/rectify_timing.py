"""Time the rectification of a 1920x1200 pair (DESIGN.md §3i): stereo_rectify, the map per camera, rectify_images end to end
(grayscale and 3 channels), and OpenCV on the host's threads for comparison; then k_rectify_map and k_remap_cubic alone under
torch.profiler in a run of its own.  Usage: python scripts/rectify_timing.py [--profile]"""
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

from multical_b200 import undistort                                    # noqa: E402
from multical_b200.camera import rectify_images, stereo_rectify        # noqa: E402
from test_gpu_rectify import make_pair                                 # noqa: E402
from test_gpu_undistort import images                                  # noqa: E402

W, H, N = 1920, 1200, 8


def best(f, reps=7):
  f()
  ts = []
  for _ in range(reps):
    t0 = time.perf_counter(); f(); ts.append(time.perf_counter() - t0)
  return min(ts) * 1e3


def main():
  import cv2
  import torch
  print(f"device: {torch.cuda.get_device_name(0)}; cv2 threads: {cv2.getNumThreads()}")
  cams, pose = make_pair("standard", W, H)
  r = stereo_rectify(*cams, pose, alpha=0.5)
  recs = [(r.R1, r.P1), (r.R2, r.P2)]
  eng = undistort.undistort_engine()
  if "--profile" in sys.argv:
    from torch.profiler import ProfilerActivity, profile
    model, vec = undistort.camera_vector(cams[0])
    src = images(np.random.default_rng(0), N, (H, W, 3))
    eng.rectify_images(model, vec, r.R1, r.P1, (W, H), src)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
      for k in range(5):
        R = r.R1.copy(); R[0, 0] += 1e-15 * (k + 1)                     # a new key: the map is computed again
        eng.rectify_map(model, vec, R, r.P1, (W, H), want_map=False)
        eng.rectify_images(model, vec, r.R1, r.P1, (W, H), src)
    for e in prof.key_averages():
      if e.key.startswith(("void mcba::k_rectify_map", "void mcba::k_remap_cubic")):
        print(f"{e.key[:60]:60s} calls {e.count:3d}  mean {e.device_time / 1e3 if hasattr(e, 'device_time') else e.cuda_time / 1e3:.3f} ms")
    return
  print(f"stereo_rectify: {best(lambda: stereo_rectify(*cams, pose, alpha=0.5)):.2f} ms")
  print(f"rectify_map (float map to host) per camera: {best(lambda: cams[0].rectify_map(*recs[0])):.2f} ms")
  for shape in ((H, W), (H, W, 3)):
    batch = [images(np.random.default_rng(1), N, shape) for _ in range(2)]
    ours = best(lambda: rectify_images(batch, cams, recs)) / (2 * N)
    maps = [cv2.initUndistortRectifyMap(c.intrinsic, c.dist, R, P, (W, H), cv2.CV_16SC2) for c, (R, P) in zip(cams, recs)]
    cvt = best(lambda: [cv2.remap(im, *maps[k], cv2.INTER_CUBIC) for k in range(2) for im in batch[k]], reps=3) / (2 * N)
    cvm = best(lambda: cv2.initUndistortRectifyMap(cams[0].intrinsic, cams[0].dist, *recs[0], (W, H), cv2.CV_32FC2), reps=3)
    print(f"{len(shape) == 3 and '3-channel' or 'grayscale'}: rectify_images {ours:.2f} ms per image end to end; "
          f"cv2.remap {cvt:.2f} ms per image, cv2.initUndistortRectifyMap {cvm:.2f} ms per camera")


if __name__ == "__main__":
  main()
