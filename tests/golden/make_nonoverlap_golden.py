"""Generate the golden vectors of the non-overlapping camera initialisation (tests/test_gpu_nonoverlap.py,
tests/test_simt_nonoverlap.py) from the UNMODIFIED reference `HandEye.initialise_camera_poses` (multical/hand_eye/hand_eye.py),
imported through tests/refshim.

Run with MULTICAL_REFERENCE pointing at a checkout of multical:
    MULTICAL_REFERENCE=<path> python tests/golden/make_nonoverlap_golden.py
Each scene stores the pose table (poses, valid, num_points), handeye_df (quads [k,4] as indices, image_ids as CSR ids/offsets, X
[k,4,4]), every (master, slave) pick of probabilistic_guess (pairs [p,2], pick index within the pair's accepted list, density), the
reference camera, cam_init [C,4,4] in camera order and the text of initial_guess.json.
"""
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "refshim"))

from multical_b200.synthetic import make_pose_table_scene  # noqa: E402
import loader  # noqa: E402


def few_images(T, valid):
  """camera 1 sees board 2 in frames 0-9 only, camera 2 in frames 8-17 only: quadruples (1, 2, 2, 2) and (2, 1, 2, 2) have 2 images."""
  F = valid.shape[1]
  valid[1, :, 2] = np.arange(F) < 10
  valid[2, :, 2] = (np.arange(F) >= 8) & (np.arange(F) < 18)
  return T, valid


def degenerate(T, valid):
  """frames 1-7 repeat frame 0 exactly and camera 0 sees board 2 in frames 0-7 only: every quadruple with (camera 0, board 2) has one
  repeated A and one repeated B, which OpenCV rejects ("determinant(R) is null"); camera 0 then has the fewest groups."""
  F = valid.shape[1]
  valid[:, 1:8] = valid[:, 0:1]
  T[:, 1:8] = T[:, 0:1]
  valid[0, :, 2] = np.arange(F) < 8
  assert valid[:, 0].all()
  return T, valid


SCENES = {
  # name: make_pose_table_scene arguments, post-processing
  "nonoverlap_all_boards": (dict(C=4, F=30, B=3, p_valid=0.8, seed=31), None),
  "nonoverlap_disjoint": (dict(C=3, F=40, B=9, p_valid=0.8, seed=32, disjoint=True), None),
  "nonoverlap_outliers": (dict(C=3, F=40, B=3, p_valid=0.9, seed=33, outliers=0.1), None),
  "nonoverlap_sparse": (dict(C=3, F=50, B=3, p_valid=0.35, seed=34), None),
  "nonoverlap_few_images": (dict(C=3, F=30, B=3, p_valid=0.9, seed=35), few_images),
  "nonoverlap_degenerate": (dict(C=3, F=30, B=3, p_valid=1.0, seed=36), degenerate),
  # 36 transforms per (master, slave) set: more than one per lane of the vote's warp
  "nonoverlap_many_boards": (dict(C=2, F=40, B=6, p_valid=0.9, seed=37), None),
}


def main():
  ref = loader.load()
  from multical.hand_eye import hand_eye
  picks = []
  orig = hand_eye.probabilistic_guess

  def recorded(transformations_list):
    density, pose = orig(transformations_list)
    idx = [k for k, t in enumerate(transformations_list) if np.array_equal(t, np.array(pose))]
    picks.append((idx[0], float(density)))
    return density, pose
  hand_eye.probabilistic_guess = recorded
  for name, (kw, post) in SCENES.items():
    picks.clear()
    T, valid, npts, cam = make_pose_table_scene(**kw)
    if post is not None:
      T, valid = post(T, valid)
    npts = np.where(valid, np.maximum(npts, 20), 0)
    names = [f"cam{c}" for c in range(valid.shape[0])]
    table = ref.Table.create(poses=T, valid=valid, num_points=npts)
    with tempfile.TemporaryDirectory() as d:
      he = hand_eye.HandEye(table, names, d)
      he.initialise_camera_poses()
      with open(os.path.join(d, "initial_guess.json")) as f:
        guess = f.read()
    df = he.handeye_df
    ids = [r["image_ids"] for r in df]
    pairs = [(m, s) for m in range(len(names)) for s in range(len(names)) if s != m]
    z = dict(poses=T, valid=valid, num_points=npts,
             quads=np.array([(names.index(r["master_cam"]), names.index(r["slave_cam"]), r["boardM"], r["boardS"]) for r in df],
                            np.int32).reshape(-1, 4),
             image_ids=np.concatenate(ids).astype(np.int64), image_start=np.concatenate([[0], np.cumsum([len(i) for i in ids])]),
             X=np.array([r["slaveCam_wrt_masterCam"] for r in df]), pairs=np.array(pairs, np.int32).reshape(-1, 2),
             pick=np.array([p[0] for p in picks], np.int32), density=np.array([p[1] for p in picks]),
             reference_camera=names.index(he.reference_camera), cam_init=np.array([he.cam_init[k] for k in names]),
             initial_guess=np.array(guess))
    np.savez_compressed(os.path.join(HERE, name + ".npz"), **z)
    n_all = sum(len(he.viewed_boards[names[m]]) * len(he.viewed_boards[names[s]]) for m, s in pairs)
    print(f"{name}: {len(df)} of {n_all} quadruples solved, reference {he.reference_camera}, set sizes "
          f"{sorted({sum(1 for r in df if (r['master_cam'], r['slave_cam']) == (names[m], names[s])) for m, s in pairs})}")


if __name__ == "__main__":
  main()
