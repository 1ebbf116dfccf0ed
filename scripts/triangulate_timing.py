"""Time triangulation (DESIGN.md §3j) on two workloads, one on each side of the group-size choice (csrc/triangulate_kernels.cuh): a
standard pair with 1 M points (groups of 2 lanes) and the cfg5 dome, 64 cameras x 2000 frames, all corners (groups of 32 lanes, 2 views
per lane).  For each: numpy-to-numpy end to end and observations per second; host arms: cv2.triangulatePoints on the pair (linear, no
distortion), the oracle (numpy + scipy, oracle/triangulate_oracle.py) on a 2000-point subsample of the dome.  With --profile: the kernels
alone under torch.profiler, in a run of their own.  Usage: python scripts/triangulate_timing.py [--profile]"""
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))

from multical_b200 import synthetic                                        # noqa: E402
from multical_b200.triangulate import triangulate, triangulate_points      # noqa: E402
from oracle import triangulate_oracle as to                                # noqa: E402
from test_gpu_triangulate import cameras_of, scene_views                   # noqa: E402


def best(f, reps=5):
  f()
  ts = []
  for _ in range(reps):
    t0 = time.perf_counter(); f(); ts.append(time.perf_counter() - t0)
  return min(ts)


def pair(n=1_000_000, seed=0):
  scene = synthetic.make_scene(C=2, F=1, seed=seed)
  g = scene["gt"]
  rng = np.random.default_rng(seed)
  X = np.stack([rng.uniform(-0.3, 0.3, n), rng.uniform(-0.2, 0.2, n), rng.uniform(0.8, 1.6, n)], 1)
  pixels = np.stack([synthetic.distort_project("standard", X @ T[:3, :3].T + T[:3, 3], g["K"][c], g["dist"][c])
                     for c, T in enumerate(g["cam_poses"])]) + rng.normal(0, 0.3, (2, n, 2))
  return scene, pixels, np.ones((2, n), bool)


def main():
  import torch
  print(f"device: {torch.cuda.get_device_name(0)}")
  scene, pixels, valid = pair()
  cams, poses = cameras_of(scene), scene["gt"]["cam_poses"]
  dome = synthetic.make_workload("cfg5")
  dpix, dvalid, _ = scene_views(dome)
  dcams, dposes = cameras_of(dome), dome["gt"]["cam_poses"]
  if "--profile" in sys.argv:
    from torch.profiler import ProfilerActivity, profile
    triangulate(cams, poses, pixels, valid); triangulate(dcams, dposes, dpix, dvalid)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
      for _ in range(3):
        triangulate(cams, poses, pixels, valid)
        triangulate(dcams, dposes, dpix, dvalid)
    for e in prof.key_averages():
      if "k_triangulate" in e.key:
        t = e.device_time if hasattr(e, "device_time") else e.cuda_time
        print(f"{e.key[:70]:70s} calls {e.count:4d}  total per call of the workload {e.count * t / 3e3:.3f} ms")
    return
  t = best(lambda: triangulate(cams, poses, pixels, valid))
  print(f"pair, 1 M points: triangulate {t * 1e3:.1f} ms end to end, {valid.sum() / t:.3g} observations/s")
  K = [c.intrinsic for c in cams]
  P = [K[c] @ poses[c, :3] for c in range(2)]
  x = [np.ascontiguousarray(pixels[c].T) for c in range(2)]
  import cv2
  tl = best(lambda: triangulate_points(P[0], P[1], x[0], x[1]))
  tc = best(lambda: cv2.triangulatePoints(P[0], P[1], x[0], x[1]), reps=3)
  print(f"pair, 1 M points: triangulate_points {tl * 1e3:.1f} ms, cv2.triangulatePoints {tc * 1e3:.1f} ms (linear only, host)")
  t = best(lambda: triangulate(dcams, dposes, dpix, dvalid), reps=3)
  print(f"cfg5 dome, {dpix.shape[1]} points, {dvalid.sum()} observations: triangulate {t * 1e3:.1f} ms end to end, "
        f"{dvalid.sum() / t:.3g} observations/s")
  idx = np.random.default_rng(0).choice(dpix.shape[1], 2000, replace=False)
  g = dome["gt"]
  t0 = time.perf_counter()
  to.triangulate(dome["model"], g["K"], g["dist"], g["cam_poses"], dpix[:, idx], dvalid[:, idx])
  to_t = time.perf_counter() - t0
  print(f"cfg5 dome, oracle on a 2000-point subsample: {to_t:.1f} s, {dvalid[:, idx].sum() / to_t:.3g} observations/s")


if __name__ == "__main__":
  main()
