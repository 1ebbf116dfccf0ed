"""CPU (-m "not gpu"): the non-overlapping camera initialisation of tests/test_gpu_nonoverlap.py on the SIMT interpreter (tests/simt)
at the sizes it runs in seconds -- both kernels and the host class, the same bars -- and oracle/nonoverlap_oracle.py against the
reference's goldens."""
import json

import numpy as np
import pytest

import test_gpu_nonoverlap as gn
from oracle import nonoverlap_oracle
from test_simt_kernels import on_the_interpreter, simt_library  # noqa: F401  (fixtures)


def test_oracle_matches_reference_golden():
  for name in gn.SCENES:
    z = gn.golden(name)
    names = gn.names_of(z)
    o = nonoverlap_oracle.initialise_camera_poses(z["poses"], z["valid"], names)
    assert o["reference_camera"] == names[int(z["reference_camera"])], name
    quads = np.array([(names.index(r["master_cam"]), names.index(r["slave_cam"]), r["boardM"], r["boardS"]) for r in o["handeye_df"]])
    assert np.array_equal(quads.reshape(-1, 4), z["quads"]), name
    assert np.abs(np.array([r["slaveCam_wrt_masterCam"] for r in o["handeye_df"]]) - z["X"]).max() < 1e-12, name
    assert np.abs(np.array([o["cam_init"][k] for k in names]) - z["cam_init"]).max() < 1e-12, name
    assert [o["sets"][tuple(p)][2] for p in z["pairs"].tolist()] == z["pick"].tolist(), name
    assert json.loads(json.dumps(o["camera_poses"])) == json.loads(str(z["initial_guess"])), name


def test_every_quadruple_matches_cv2():
  gn.run_quads_against_cv2([3, 4, 5, 7, 31, 128, 129, 300] + [12] * 10, degenerate_reps=2)


def test_vote_matches_gaussian_kde():
  gn.run_vote_against_scipy([4, 4, 5, 7, 32, 33, 70])


@pytest.mark.parametrize("name", gn.SCENES)
def test_initialise_camera_poses_matches_reference_golden(name):
  gn.run_golden(name)


def test_bit_reproducible():
  gn.run_reproducible("nonoverlap_disjoint")


def test_files_written_only_with_an_image_path(tmp_path, monkeypatch):
  gn.run_files(tmp_path, monkeypatch)


test_reference_failures_raise_value_error = gn.test_reference_failures_raise_value_error
test_bad_inputs = gn.test_bad_inputs
