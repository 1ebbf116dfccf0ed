"""CPU (-m "not gpu"): the checks of tests/test_gpu_rectify.py on the SIMT interpreter (tests/simt) at small sizes, and the numpy
restatement of OpenCV's row walk (oracle/rectify_oracle.py) against live cv2 on random R and P, at widths that are not multiples of 8,
and at R = I, P = K (the undistortion map)."""
import numpy as np
import pytest

import test_gpu_rectify as gr
import test_gpu_undistort as gu
from multical_b200 import undistort
from oracle import rectify_oracle as ro
from test_simt_kernels import on_the_interpreter, simt_library  # noqa: F401  (fixtures)


@pytest.fixture(autouse=True)
def fresh_undistort_engines(on_the_interpreter, monkeypatch):  # noqa: F811
  monkeypatch.setattr(undistort, "_engines", {})
  yield
  for eng in undistort._engines.values(): eng.close()


def test_oracle_walk_is_opencvs():
  import cv2
  rng = np.random.default_rng(4)
  for k, (w, h) in enumerate([(97, 61), (64, 48), (101, 37), (13, 9), (7, 5)]):
    for model in gr.MODELS:
      cams, _ = gr.make_pair(model, w, h, skew=1.5 * (k % 2), seed=k)
      K, d = cams[0].intrinsic, cams[0].dist
      R = cv2.Rodrigues(rng.normal(0, 0.08, 3))[0]
      P = np.array([[K[0, 0] * rng.uniform(0.8, 1.2), 0, rng.uniform(0.3, 0.7) * w, 0],
                    [0, K[1, 1] * rng.uniform(0.8, 1.2), rng.uniform(0.3, 0.7) * h, 0], [0, 0, 1, 0]])
      size = (w + k, h)
      ref = gr.cv_map(cams[0], R, P, size)
      ours = ro.rectify_map(K, d, R, P, size, fisheye=model == "fisheye")
      assert np.array_equal(ours.view(np.int32), ref.view(np.int32)), (model, w, h)
  for model in gr.MODELS:
    for skew in (0.0, 2.5):
      cam = gu.make_camera(model, 97, 61, skew=skew)
      ours = ro.rectify_map(cam.intrinsic, cam.dist, np.eye(3), cam.intrinsic, cam.image_size, fisheye=model == "fisheye")
      assert np.array_equal(ours.view(np.int32), gu.cv_map(cam).view(np.int32)), (model, skew)


def test_stereo_rectify_matches_opencv():
  gr.run_stereo_rectify(64, 48)


def test_stereo_rectify_fisheye_matches_opencv():
  gr.run_stereo_rectify_fisheye(64, 48)


def test_maps_are_opencvs_bit_for_bit():
  gr.run_maps([(64, 48), (37, 23)])


def test_wide_maps_are_opencvs_bit_for_bit():
  gr.run_wide_maps()


def test_rectify_images_are_cv2_remap_bit_for_bit():
  gr.run_images(48, 36)


def test_rectify_points_match_opencv():
  gr.run_points(64, 48, 200)


def test_calibrated_pair_rectifies_to_equal_rows():
  gr.run_end_to_end(F=6)


def test_repeated_calls_agree_bit_for_bit():
  gr.run_reproducible(40, 30)


def test_refusals():
  gr.run_errors(16, 12)
