"""CPU (-m "not gpu"): the checks of tests/test_gpu_undistort.py on the SIMT interpreter (tests/simt) at small sizes, the device's bicubic
weight table entry by entry against the recipe restated in oracle/undistort_oracle.py, and that restatement against live cv2.remap."""
import numpy as np
import pytest

import test_gpu_undistort as gu
from multical_b200 import undistort
from oracle import undistort_oracle as uo
from test_simt_kernels import on_the_interpreter, simt_library  # noqa: F401  (fixtures)


@pytest.fixture(autouse=True)
def fresh_undistort_engines(on_the_interpreter, monkeypatch):  # noqa: F811
  monkeypatch.setattr(undistort, "_engines", {})
  yield
  for eng in undistort._engines.values(): eng.close()


def test_cubic_table_is_the_recipe():
  dev = undistort.undistort_engine().remap_cubic_table()
  ref = uo.cubic_table()
  assert np.array_equal(dev, ref), f"{int((dev != ref).any(axis=1).sum())} table entries differ"
  assert (ref.sum(axis=1) == 1 << 15).all()


def test_oracle_remap_is_cv2_remap():
  """The restated recipe against cv2.remap on random maps, with exact half-way positions and windows up to 5 px outside the image."""
  import cv2
  rng = np.random.default_rng(2)
  for shape in [(60, 80), (60, 80, 3), (45, 70), (90, 101, 3)]:
    src = rng.integers(0, 256, shape, dtype=np.uint8)
    m = (rng.random((60, 80, 2)) * [shape[1] + 10, shape[0] + 10] - 5).astype(np.float32)
    m[::3] = (np.floor(m[::3] * 32) + 0.5) / 32                      # ties: rint goes to even
    assert np.array_equal(uo.remap_cubic(src, m), cv2.remap(src, m, None, cv2.INTER_CUBIC)), shape


def test_oracle_map_is_opencvs():
  for model in gu.MODELS:
    cam = gu.make_camera(model, 97, 61, skew=2.5)
    ref = gu.cv_map(cam)
    assert np.array_equal(uo.undistort_map(cam.intrinsic, cam.dist, cam.image_size, fisheye=model == "fisheye").view(np.int32),
                          ref.view(np.int32)), model


def test_maps_are_opencvs_bit_for_bit():
  gu.run_maps([(64, 48), (37, 23)])


def test_remap_is_cv2_remap_bit_for_bit():
  gu.run_remap(64, 48)


def test_undistort_images_match_reference_per_image_remap():
  gu.run_undistort_images([(64, 48), (37, 23), (50, 40)], 2)


def test_project_and_undistort_points_match_opencv():
  gu.run_points(64, 48, 200)


def test_repeated_calls_agree_bit_for_bit():
  gu.run_reproducible(40, 30)


def test_unsupported_images_raise():
  gu.run_errors(16, 12)
