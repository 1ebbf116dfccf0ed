"""Time the pose-graph initialisation (multical_b200.tables.initialise_poses) at the BASELINE shapes cfg2..cfg5 on synthetic pose tables,
with oracle/pose_init_oracle.py (numpy + scipy, the reference's algorithm) on the same host next to it.

    python scripts/pose_init_timing.py [cfg2 cfg3 ...] [--no-oracle]
Prints the card name and power limit, then per shape: end-to-end time of initialise_poses (median of 3 after a warm-up), device time of
each entry (CUDA events around mcba_pose_pairs for both axes and mcba_pose_times), and the oracle's host time."""
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from multical_b200 import synthetic, tables  # noqa: E402
from multical_b200.calibration import get_engine  # noqa: E402
from multical_b200.structs import Table  # noqa: E402
from oracle import pose_init_oracle  # noqa: E402

SHAPES = dict(cfg2=(4, 200, 1, 0.9), cfg3=(8, 500, 1, 0.9), cfg4=(16, 1000, 5, 0.5), cfg5=(64, 2000, 1, 0.9))


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
    tables.initialise_poses(table)
    ts = []
    for _ in range(3):
      t0 = time.perf_counter(); out = tables.initialise_poses(table); ts.append(time.perf_counter() - t0)
    cam_pairs = tables.select_pairs(tables.pattern_overlaps(valid, npts, 0))[1]
    board_pairs = tables.select_pairs(tables.pattern_overlaps(valid, npts, 2))[1]
    d_cam = device_ms(lambda: eng.pose_pairs(poses, valid, 0, cam_pairs)) if cam_pairs else 0.0
    d_board = device_ms(lambda: eng.pose_pairs(poses, valid, 2, board_pairs)) if board_pairs else 0.0
    d_times = device_ms(lambda: eng.pose_times(poses, valid, out.camera.poses, out.camera.valid, out.board.poses, out.board.valid))
    line = (f"{name} C={C} F={F} B={B}: initialise_poses {1e3 * np.median(ts):.1f} ms (min {1e3 * min(ts):.1f}); "
            f"mcba_pose_pairs cameras {d_cam:.2f} ms, boards {d_board:.2f} ms; mcba_pose_times {d_times:.2f} ms")
    if "--no-oracle" not in sys.argv:
      t0 = time.perf_counter(); pose_init_oracle.initialise_poses(poses, valid, npts); line += f"; oracle (host) {time.perf_counter() - t0:.2f} s"
    print(line, flush=True)


if __name__ == "__main__":
  main()
