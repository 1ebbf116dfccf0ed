"""Generate the golden vectors of the pose-graph initialisation (tests/test_gpu_pose_init.py, tests/test_simt_pose_init.py) from the
UNMODIFIED reference `tables.initialise_poses` (multical/tables.py:354-377), imported through tests/refshim.

Run with MULTICAL_REFERENCE pointing at a checkout of multical:
    MULTICAL_REFERENCE=<path> python tests/golden/make_pose_init_golden.py
Each scene stores the pose table (poses, valid, num_points), the optional camera_poses, what initialise_poses returns (camera, board,
times: poses and valid), the masters and pairs of both axes, and every align_transforms_robust call (m1, m2, valid -> t, inliers),
recorded by wrapping the reference's function, as call_<k>_{m1,m2,valid,t,inliers}.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "refshim"))

from multical_b200.synthetic import make_pose_table_scene as pose_table  # noqa: E402
import loader  # noqa: E402


SCENES = {
  # name: pose_table(...) arguments, camera_poses given
  "pose_init_arc": (dict(C=4, F=30, B=1, p_valid=0.9, seed=11), False),
  "pose_init_cube": (dict(C=3, F=12, B=5, p_valid=0.7, seed=12), False),
  "pose_init_outliers": (dict(C=3, F=40, B=2, p_valid=0.9, seed=13, outliers=0.15), False),
  # rows of 1, 2, 3 (frames: C x B with cameras missing), 29, 30, 31 (camera pairs: F*B rows)
  "pose_init_rows_29": (dict(C=3, F=29, B=1, p_valid=1.0, seed=14), False),
  "pose_init_rows_30": (dict(C=2, F=30, B=1, p_valid=1.0, seed=15), False),
  "pose_init_rows_31": (dict(C=3, F=31, B=1, p_valid=0.97, seed=16), False),
  "pose_init_sparse": (dict(C=3, F=20, B=1, p_valid=0.4, seed=17), False),
  "pose_init_dead_camera": (dict(C=4, F=24, B=1, p_valid=0.9, seed=18, dead_camera=3, empty_frame=5), False),
  "pose_init_camera_poses": (dict(C=3, F=20, B=2, p_valid=0.8, seed=19), True),
  # a board pair of C*F = 1040 rows: above the 1024-row small/large switch (only the calls of 1000 rows or more are recorded)
  "pose_init_large": (dict(C=2, F=520, B=2, p_valid=0.9, seed=20, outliers=0.05), False),
}
MIN_RECORDED_ROWS = {"pose_init_large": 1000}


class _Indexer:
  """py-structs lets tables.py both call and subscript `Table._index` (tables.py:104-110, 114-121); the shim only calls it.  Installed
  on the shim's Table in this process alone, so tests/golden/make_golden.py keeps the shim as it is."""
  def __init__(self, table, index): self.table, self.index = table, index
  def __call__(self, idx): return self.index(self.table, idx)
  def __getitem__(self, idx): return self.index(self.table, idx)


def main():
  ref = loader.load()
  from structs import numpy as shim_numpy
  shim_numpy.Table._index = property(lambda self: _Indexer(self, shim_numpy._index))
  from multical import tables
  from multical.transform import matrix
  calls = []
  orig = matrix.align_transforms_robust

  def recorded(m1, m2, valid=None, threshold=1.5):
    t, inliers = orig(m1, m2, valid, threshold)
    calls.append((np.array(m1), np.array(m2), np.ones(len(m1), bool) if valid is None else np.array(valid), t, inliers))
    return t, inliers
  matrix.align_transforms_robust = recorded
  pairs = {}
  orig_select = tables.graph.select_pairs

  def select(overlaps, hop_penalty=0.8):
    master, p = orig_select(overlaps, hop_penalty)
    pairs.setdefault("list", []).append((master, list(p)))
    return master, p
  tables.graph.select_pairs = select
  for name, (kw, with_cam) in SCENES.items():
    calls.clear(); pairs.clear()
    T, valid, npts, cam = pose_table(**kw)
    table = ref.Table.create(poses=T, valid=valid, num_points=npts)
    cam_poses = cam @ np.linalg.inv(cam[0]) if with_cam else None
    out = tables.initialise_poses(table, camera_poses=cam_poses)
    (cm, cp), (bm, bp) = pairs["list"]
    z = dict(poses=T, valid=valid, num_points=npts, has_camera_poses=with_cam,
             camera_poses=cam_poses if with_cam else np.zeros((0, 4, 4)),
             camera=out.camera.poses, camera_valid=out.camera.valid, board=out.board.poses, board_valid=out.board.valid,
             times=out.times.poses, times_valid=out.times.valid, camera_master=cm, camera_pairs=np.array(cp, np.int32).reshape(-1, 2),
             board_master=bm, board_pairs=np.array(bp, np.int32).reshape(-1, 2), n_calls=len(calls))
    calls[:] = [c for c in calls if len(c[0]) >= MIN_RECORDED_ROWS.get(name, 0)]
    z["n_calls"] = len(calls)
    for k, (m1, m2, v, t, inl) in enumerate(calls):
      z.update({f"call_{k}_m1": m1, f"call_{k}_m2": m2, f"call_{k}_valid": v, f"call_{k}_t": t, f"call_{k}_inliers": inl})
    np.savez_compressed(os.path.join(HERE, name + ".npz"), **z)
    sizes = sorted({len(c[0]) for c in calls})
    print(f"{name}: {len(calls)} calls, rows {sizes[:6]}..{sizes[-1]}, inliers rejected {sum(int((c[2] & ~c[4]).sum()) for c in calls)}")


if __name__ == "__main__":
  main()
