"""Time the exact trust-region step (`tr_solver="exact"`) against the default subspace step on the GPU.

  python scripts/exact_tr_timing.py [--repeats R] [--out DIR]

Per case and mode: device time per solve (the engine's CUDA-event time of mcba_solve, median of R solves after one warm-up), nfev,
LM iterations (accepted steps), alpha iterations per LM iteration (mcba_last_alpha_iterations / iterations) and the final cost.
Cases: bench.py's cfg2 and cfg4 scenes (bundle adjustment with bench.py's solve options) and a 50-view rational camera (the intrinsic
solve of tests/test_gpu_exact_trust_region.py, tolerances 1e-15).  The GPU's name, power limit and SM clock are printed with the numbers."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from multical_b200 import intrinsics, synthetic  # noqa: E402
from multical_b200.calibration import from_scene  # noqa: E402

BA_KW = dict(ftol=1e-4, max_nfev=100)        # bench.py's solve options (Calibration.bundle_adjust defaults)


def gpu_info():
  q = "name,power.limit,clocks.max.sm,clocks.sm"
  return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()


def summary(infos):
  ms = sorted(i.device_ms for i in infos)
  last = infos[-1]
  iters = max(len(last.log) - 1, 1)
  return dict(device_ms=ms[len(ms) // 2], nfev=last.nfev, lm_iterations=len(last.log) - 1,
              alpha_iterations_per_lm_iteration=last.alpha_iterations / iters, cost=last.cost, status=last.status)


def bundle_case(name, repeats):
  scene = synthetic.make_workload(name, seed=0)
  calib = from_scene(scene).enable(cameras=True)
  state0 = calib._state_arrays()
  eng = calib._upload(calib.inliers)
  out = {}
  for mode in ("lsmr", "exact"):
    infos = []
    for _ in range(repeats + 1):
      eng.set_params(*state0)
      infos.append(eng.solve(tr_solver=mode, **BA_KW))
    out[mode] = summary(infos[1:])
  return out


def rational_case(repeats):
  import test_gpu_exact_trust_region as et
  board, views = et.valley_views("rational")
  tight = dict(ftol=1e-15, xtol=1e-15, gtol=1e-15, max_nfev=500)
  out = {}
  for mode in ("lsmr", "exact"):
    infos = [intrinsics.calibrate_views([board], [views], [(et.W, et.H)], model="rational", tr_solver=mode, **tight)[0].solve
             for _ in range(repeats + 1)]
    out[mode] = summary(infos[1:])
  return out


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--repeats", type=int, default=5)
  ap.add_argument("--out", default=None)
  args = ap.parse_args()
  res = dict(gpu=gpu_info(), cfg2=bundle_case("cfg2", args.repeats), cfg4=bundle_case("cfg4", args.repeats),
             rational_50_views=rational_case(args.repeats))
  print(json.dumps(res, indent=1))
  if args.out:
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "exact_tr_timing.json"), "w") as f: json.dump(res, f, indent=1)


if __name__ == "__main__":
  main()
