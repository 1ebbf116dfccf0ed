"""Time undistort_images (multical_b200/undistort.py) on the GPU against the reference's undistort_images (cv2.remap INTER_CUBIC over a
thread pool, camera.py:244-258) on the same host, at the cfg4 rig shape: 16 cameras x N views of 1920 x 1200 seeded synthetic grayscale
images, plus one camera of 3-channel images.

  python scripts/undistort_timing.py [--out DIR] [--cameras 16] [--views N] [--width 1920] [--height 1200]

  maps         host clock around undistort_map for every camera (computed on the device, copied back as float32 [h, w, 2])
  kernel       device time of k_remap_cubic per image from torch.profiler (CUDA activities), in a run of its own; achieved bytes/s over
               the algorithmic bytes: W*H*ch read + W*H*ch written, and with the resident map's 6 bytes per pixel that the kernel reads
               for every image
  copies       the host<->device copies of that run, per image
  end_to_end   host clock around undistort_images from nested numpy lists to nested numpy lists (maps resident from the warm-up)
  reference    the reference's undistort_images restated: cv2.remap(image, camera.undistort_map, None, INTER_CUBIC) over
               ThreadPool(cpu_count()).imap(chunksize=4), maps from cv2.initUndistortRectifyMap, on this host's CPU
The outputs are compared with cv2.remap at the timed size.  The GPU's name, power limit and SM clocks are printed with the numbers."""
import argparse
import json
import os
import sys
import time
from multiprocessing import cpu_count
from multiprocessing.pool import ThreadPool

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from intrinsics_timing import gpu_info  # noqa: E402
from multical_b200 import undistort  # noqa: E402
from multical_b200.camera import Camera, undistort_images  # noqa: E402

MAP_BYTES_PER_PIXEL = 6


def rig(C, w, h, seed=0):
  rng = np.random.default_rng(seed)
  cams = []
  for _ in range(C):
    f = rng.uniform(1300, 1500)
    K = np.array([[f, 0, w / 2 + rng.uniform(-20, 20)], [0, f * rng.uniform(0.995, 1.005), h / 2 + rng.uniform(-20, 20)], [0, 0, 1]])
    d = np.array([rng.uniform(-0.3, -0.1), rng.uniform(0.0, 0.15), rng.uniform(-1e-3, 1e-3), rng.uniform(-1e-3, 1e-3), rng.uniform(-0.05, 0.0)])
    cams.append(Camera(image_size=(w, h), intrinsic=K, dist=d))
  return cams


def make_images(rng, n, shape):
  h, w = shape[:2]
  yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
  base = 128 + 100 * np.sin(xx / 17.0) * np.cos(yy / 23.0)
  if len(shape) == 3: base = base[..., None] + np.array([-30, 0, 30], np.float32)
  return [np.clip(base + rng.normal(0, 20, shape).astype(np.float32), 0, 255).astype(np.uint8) for _ in range(n)]


def reference_undistort_images(images, maps, j=cpu_count(), chunksize=4):
  import cv2
  with ThreadPool(processes=j) as pool:
    pairs = [(image, m) for m, cam_images in zip(maps, images) for image in cam_images]
    out = list(pool.imap(lambda a: cv2.remap(a[0], a[1], None, cv2.INTER_CUBIC), pairs, chunksize=chunksize))
  sizes = np.cumsum([0] + [len(i) for i in images])
  return [out[a:b] for a, b in zip(sizes[:-1], sizes[1:])]


def profile_kernels(batch, cams):
  import torch
  from torch.profiler import ProfilerActivity, profile
  with profile(activities=[ProfilerActivity.CUDA]) as prof:
    undistort_images(batch, cams)
    torch.cuda.synchronize()
  kern, h2d, d2h = [], [], []
  for e in prof.events():
    if e.device_type.name != "CUDA": continue
    t = e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
    if "k_remap_cubic" in e.name: kern.append(t)
    elif "HtoD" in e.name: h2d.append(t)
    elif "DtoH" in e.name: d2h.append(t)
  return kern, h2d, d2h


def time_case(name, cams, batch, repeats=3):
  n_img = sum(len(b) for b in batch)
  h, w = batch[0][0].shape[:2]
  ch = 1 if batch[0][0].ndim == 2 else batch[0][0].shape[2]
  t = time.perf_counter()
  for c in cams: c.__dict__.pop("undistort_map", None); _ = c.undistort_map
  maps_ms = 1e3 * (time.perf_counter() - t)
  out = undistort_images(batch, cams)                                  # warm-up: maps resident, staging allocated
  e2e = []
  for _ in range(repeats):
    t = time.perf_counter()
    out = undistort_images(batch, cams)
    e2e.append(1e3 * (time.perf_counter() - t))
  # correctness at the timed size: every camera's first and last image against cv2.remap on OpenCV's map
  import cv2
  bad = 0
  cv_maps = [cv2.initUndistortRectifyMap(c.intrinsic, c.dist, None, c.intrinsic, c.image_size, cv2.CV_32FC2)[0] for c in cams]
  for m, ims, outs in zip(cv_maps, batch, out):
    for i in (0, len(ims) - 1):
      bad += int((cv2.remap(ims[i], m, None, cv2.INTER_CUBIC) != outs[i]).sum())
  try:
    kern, h2d, d2h = profile_kernels(batch, cams)
  except Exception as e:                                               # the other numbers stand without the profile
    print(f"profile failed: {e!r}", file=sys.stderr)
    kern, h2d, d2h = [float("nan")], [float("nan")], [float("nan")]
  kern_us = float(np.sum(kern))
  px = w * h
  per_image_kernel_us = kern_us / n_img
  algo = 2 * px * ch
  ref = []
  for _ in range(repeats):
    t = time.perf_counter()
    reference_undistort_images(batch, cv_maps)
    ref.append(1e3 * (time.perf_counter() - t))
  return dict(case=name, cameras=len(cams), images=n_img, size=[w, h], channels=ch, maps_ms=maps_ms,
              kernel_us_per_image=per_image_kernel_us, kernel_launches=len(kern),
              achieved_GBps_image_bytes=algo / per_image_kernel_us * 1e-3,
              achieved_GBps_with_map=(algo + MAP_BYTES_PER_PIXEL * px) / per_image_kernel_us * 1e-3,
              h2d_us_per_image=float(np.sum(h2d)) / n_img, d2h_us_per_image=float(np.sum(d2h)) / n_img,
              end_to_end_ms=e2e, end_to_end_ms_per_image=min(e2e) / n_img,
              reference_ms=ref, reference_ms_per_image=min(ref) / n_img, host_threads=cpu_count(), cv2=cv2.__version__,
              pixels_differing_from_cv2=bad)


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--out", default=None)
  ap.add_argument("--cameras", type=int, default=16)
  ap.add_argument("--views", type=int, default=20)
  ap.add_argument("--width", type=int, default=1920)
  ap.add_argument("--height", type=int, default=1200)
  args = ap.parse_args()
  results = [dict(gpu=gpu_info())]
  rng = np.random.default_rng(1)
  cams = rig(args.cameras, args.width, args.height)
  gray = [make_images(rng, args.views, (args.height, args.width)) for _ in cams]
  results.append(time_case(f"cfg4_{args.cameras}x{args.views}_gray", cams, gray))
  del gray
  color = [make_images(rng, args.views, (args.height, args.width, 3))]
  results.append(time_case(f"one_camera_{args.views}_bgr", cams[:1], color))
  results.append(dict(gpu_after=gpu_info()))
  for r in results: print(json.dumps(r))
  if args.out:
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "undistort_timing.json"), "w") as fh:
      json.dump(results, fh, indent=1)


if __name__ == "__main__":
  main()
