"""TEST INFRASTRUCTURE ONLY — import the unmodified reference hot path from a checkout of multical whose
location is given by the MULTICAL_REFERENCE environment variable.  Only tests/golden/make_golden.py uses it:
the test-suite compares against the golden vectors it stores, never against the reference itself.

Recipe = SURVEY.md Appendix B: stand-in `structs`, `cached_property` alias, empty
`quaternion`, and stub *packages* for `multical` / `multical.board` whose __path__ points
at the reference tree so its heavy __init__.py files (omegaconf, Qt, ...) are skipped.
"""
import functools
import os
import sys
import types

REFERENCE_ROOT = os.environ.get("MULTICAL_REFERENCE", "")


def available():
  return bool(REFERENCE_ROOT) and os.path.isdir(os.path.join(REFERENCE_ROOT, "multical"))


def load():
  """Returns a namespace with the reference classes; raises if the reference is absent."""
  if not available():
    raise RuntimeError("set MULTICAL_REFERENCE to a checkout of multical")
  here = os.path.dirname(os.path.abspath(__file__))
  if here not in sys.path:
    sys.path.insert(0, here)
  if "cached_property" not in sys.modules:
    m = types.ModuleType("cached_property")
    m.cached_property = functools.cached_property
    sys.modules["cached_property"] = m
  sys.modules.setdefault("quaternion", types.ModuleType("quaternion"))
  for name, sub in (("multical", ""), ("multical.board", "/board")):
    if name not in sys.modules:
      p = types.ModuleType(name)
      p.__path__ = [REFERENCE_ROOT + "/multical" + sub]
      sys.modules[name] = p

  from multical.optimization.calibration import Calibration, select_threshold
  from multical.optimization.parameters import ParamList, Parameters
  from multical.optimization.pose_set import PoseSet
  from multical.motion.static_frames import StaticFrames
  from multical.camera import Camera
  from multical.camera_fisheye import CameraFisheye
  from multical.board.board import Board
  from multical import tables
  from structs.numpy import Table
  from structs.struct import struct
  import numpy as np

  class SyntheticBoard(Parameters, Board):
    """Board exposing exactly what the hot path reads (tables.py:385-394,
    board/charuco.py:112-117): adjusted_points, num_points, params/with_params."""
    def __init__(self, adjusted_points):
      self.adjusted_points = adjusted_points
    @property
    def points(self): return self.adjusted_points
    @property
    def num_points(self): return self.adjusted_points.shape[0]
    @functools.cached_property
    def params(self): return self.adjusted_points
    def with_params(self, params): return SyntheticBoard(params)

  return types.SimpleNamespace(
    Calibration=Calibration, select_threshold=select_threshold, ParamList=ParamList,
    Parameters=Parameters, PoseSet=PoseSet, StaticFrames=StaticFrames, Camera=Camera,
    CameraFisheye=CameraFisheye, Board=Board, SyntheticBoard=SyntheticBoard,
    tables=tables, Table=Table, struct=struct)


def build_calibration(ref, scene, guess=True, motion=None):
  """Reference Calibration from a multical_b200.synthetic scene dict (plain numpy).
  motion: None -> StaticFrames over the scene's frame poses; ("rolling", end_poses) -> RollingFrames with the scene's frame poses
  as start poses; ("hand_eye", base_wrt_gripper, world_wrt_base, gripper_wrt_camera) -> HandEye."""
  import numpy as np
  s = scene
  src = s["init"] if guess else s["gt"]
  Cam = ref.CameraFisheye if s["model"] == "fisheye" else ref.Camera
  cams = []
  for i in range(s["C"]):
    kw = {} if s["model"] == "fisheye" else dict(model=s["model"])
    cams.append(Cam(image_size=tuple(s["image_size"]), intrinsic=src["K"][i].copy(),
                    dist=src["dist"][i].copy(), **kw))
  cam_names = [f"cam{i}" for i in range(s["C"])]
  boards = [ref.SyntheticBoard(p.copy()) for p in s["board_points"]]
  board_names = [f"board{i}" for i in range(len(boards))]
  pt = ref.Table.create(points=s["points"].copy(), valid=s["valid"].copy())
  def pose_table(T, valid): return ref.Table.create(poses=T.copy(), valid=valid.copy())
  calib = ref.Calibration(
    ref.ParamList(cams, cam_names), ref.ParamList(boards, board_names), pt,
    ref.PoseSet(pose_table(src["cam_poses"], s["cam_valid"]), cam_names),
    ref.PoseSet(pose_table(src["board_poses"], s["board_valid"]), board_names),
    _motion_model(ref, motion, src, s, pose_table))
  return calib


def _motion_model(ref, motion, src, s, pose_table):
  if motion is None:
    return ref.StaticFrames(pose_table(src["frame_poses"], s["frame_valid"]), None)
  names = [str(i) for i in range(s["F"])]
  if motion[0] == "rolling":
    from multical.motion.rolling_frames import RollingFrames
    return RollingFrames(src["frame_poses"].copy(), motion[1].copy(), s["frame_valid"].copy(), names)
  if motion[0] == "hand_eye":
    from multical.motion.hand_eye import HandEye
    return HandEye(pose_table(motion[1], s["frame_valid"]), motion[2].copy(), motion[3].copy(), names)
  raise ValueError(motion)
