import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
  sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")
GOLDEN_CASES = ["standard_2x6", "fisheye_3x5", "rational_2x5", "cube3_3x6", "poses_only_2x6", "invalid_poses_3x6",
                "thin_prism_2x5", "tilted_2x5"]


def pytest_configure(config):
  config.addinivalue_line("markers", "gpu: needs an H100 (sm_90a); run with -m gpu on a machine that has one")


def load_golden(name):
  """Golden fixture -> (scene dict shaped like multical_b200.synthetic scenes, raw npz dict)."""
  z = dict(np.load(os.path.join(GOLDEN, name + ".npz"), allow_pickle=False))
  C, F, B, P = z["valid"].shape
  src = dict(K=z["K"], dist=z["dist"], cam_poses=z["cam_poses"], frame_poses=z["frame_poses"], board_poses=z["board_poses"])
  scene = dict(C=C, F=F, B=B, P=P, model=str(z["model"]), image_size=tuple(int(v) for v in z["image_size"]),
               board_points=[bp for bp in z["board_points"]], points=z["points"], valid=z["valid"],
               cam_valid=z["cam_valid"], frame_valid=z["frame_valid"], board_valid=z["board_valid"], init=src, gt=src)
  return scene, z


def optimize_of(z):
  return dict(cameras=bool(z["cameras_enabled"]))


@pytest.fixture(scope="session")
def build_lib():
  import __graft_entry__ as g
  g.build()
  return g
