"""Time the non-overlapping camera initialisation (multical_b200.nonoverlap.HandEye.initialise_camera_poses) at the cfg4 shape and a
large rig on synthetic pose tables, with oracle/nonoverlap_oracle.py (the reference's algorithm: cv2 and scipy) on the same host.

    python scripts/nonoverlap_timing.py [cfg4 large] [--no-oracle]
Prints the card name and power limit, then per shape: end-to-end time of initialise_camera_poses (median of 3 after a warm-up), the
time of each entry (CUDA events around mcba_hand_eye_quads and mcba_hand_eye_vote, uploads and downloads included), and the oracle's
host time.  The oracle solves a random subsample of ORACLE_SAMPLE quadruples and the time is extrapolated to all of them; its vote
(one gaussian_kde per camera pair) is timed in full."""
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from multical_b200 import synthetic  # noqa: E402
from multical_b200.calibration import get_engine  # noqa: E402
from multical_b200.nonoverlap import HandEye  # noqa: E402
from multical_b200.structs import Table  # noqa: E402
from oracle import nonoverlap_oracle  # noqa: E402

SHAPES = dict(cfg4=(16, 1000, 5, 0.5), large=(64, 2000, 4, 0.5))
ORACLE_SAMPLE = 300


def device_ms(fn):
  a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  torch.cuda.synchronize(); a.record(); fn(); b.record(); b.synchronize()
  return a.elapsed_time(b)


def main():
  names = [a for a in sys.argv[1:] if a in SHAPES] or list(SHAPES)
  q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
  print(f"device: {q.stdout.strip()}", flush=True)
  torch.cuda.init()
  eng = get_engine()
  for name in names:
    C, F, B, p = SHAPES[name]
    poses, valid, npts, _ = synthetic.make_pose_table_scene(C, F, B, p, seed=1)
    table = Table.create(poses=poses, valid=valid, num_points=npts)
    cams = [f"cam{c}" for c in range(C)]
    HandEye(table, cams).initialise_camera_poses()
    ts = []
    for _ in range(3):
      t0 = time.perf_counter(); he = HandEye(table, cams); he.initialise_camera_poses(); ts.append(time.perf_counter() - t0)
    quads = np.array(he.quadruples(), np.int32)
    d_quads = device_ms(lambda: eng.hand_eye_quads(poses, valid, quads))
    X, _, _, ok = eng.hand_eye_quads(poses, valid, quads)
    pair = quads[:, 0] * C + quads[:, 1]
    sets = [X[ok & (pair == k)][:, :3, 3] for k in np.unique(pair)]
    d_vote = device_ms(lambda: eng.hand_eye_vote(sets))
    line = (f"{name} C={C} F={F} B={B}: {len(quads)} quadruples, {int(ok.sum())} solved; initialise_camera_poses "
            f"{1e3 * np.median(ts):.1f} ms (min {1e3 * min(ts):.1f}); mcba_hand_eye_quads {d_quads:.2f} ms; mcba_hand_eye_vote {d_vote:.2f} ms")
    if "--no-oracle" not in sys.argv:
      sample = np.random.default_rng(0).choice(len(quads), min(ORACLE_SAMPLE, len(quads)), replace=False)
      t0 = time.perf_counter()
      for k in sample:
        nonoverlap_oracle.master_slave_pair(poses, valid, *quads[k])
      solves = (time.perf_counter() - t0) * len(quads) / len(sample)
      t0 = time.perf_counter()
      for s in sets:
        nonoverlap_oracle.kde_vote(s)
      votes = time.perf_counter() - t0
      line += f"; oracle (host) {solves + votes:.1f} s ({len(sample)} solves timed and extrapolated, votes {votes:.2f} s)"
    print(line, flush=True)


if __name__ == "__main__":
  main()
