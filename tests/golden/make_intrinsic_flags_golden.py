"""Generate the golden vectors of the intrinsic calibration with OpenCV calibration flags (tests/test_gpu_intrinsic_flags.py) from the
UNMODIFIED reference `Camera.calibrate(..., flags=...)` (multical/camera.py:68-105), imported through tests/refshim.

Run with MULTICAL_REFERENCE pointing at a checkout of multical:
    MULTICAL_REFERENCE=<path> python tests/golden/make_intrinsic_flags_golden.py
Each case is a scene of make_intrinsics_golden.py's kind (the same fields: detections, arguments, K, dist, err, error_perview,
board_ids, image_ids, rounds) plus `flags`, the value the reference ORs into OpenCV's flags.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import make_intrinsics_golden as base  # noqa: E402

CALIB_FIX_K3 = 128
LOOP_40 = dict(scene=dict(C=1, F=40, vis=0.4, seed=65), outliers={3: 4.0, 17: 4.0, 29: 2.0, 8: 2.0, 33: 1.0, 12: 1.0}, limit=0.6)
CASES = {
  # the multi-round scene of intrinsics_loop_40 with k3 held at zero, at the reference's default criteria (10, 1e-3): there OpenCV stops
  # at RMS 0.5455, 1.2 % in fx away from the minimum (0.5346) that it reaches with (500, 1e-15)
  "intrinsic_flags_loop_40": dict(LOOP_40, kw=dict(model="standard", flags=CALIB_FIX_K3)),
  # the same call with the reference's max_iter / eps raised so that OpenCV reaches that minimum
  "intrinsic_flags_loop_40_tight": dict(LOOP_40, kw=dict(model="standard", flags=CALIB_FIX_K3, max_iter=500, eps=1e-15)),
}


def main(names):
  ref = base.loader.load()
  for n in names or CASES:
    spec = CASES[n]
    base.make_case(ref, n, spec)
    path = os.path.join(HERE, f"{n}.npz")
    z = dict(np.load(path, allow_pickle=False))
    z["flags"] = np.int64(spec["kw"]["flags"])
    z["max_iter"], z["eps"] = np.int64(spec["kw"].get("max_iter", 10)), np.float64(spec["kw"].get("eps", 1e-3))
    np.savez_compressed(path, **z)
    print(n, "flags", int(z["flags"]), "dist", z["dist"].ravel())


if __name__ == "__main__":
  main(sys.argv[1:])
