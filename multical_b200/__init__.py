"""multical_b200 — H100-native (sm_90a) bundle-adjustment engine behind multical's `Calibration.bundle_adjust()`.

Only the hot path of the reference (multical/optimization/calibration.py:199-212) lives here:
  csrc/         hand-written sm_90a CUDA kernels + the C-ABI (include/mcba.h) -> libmcba.so
  engine.py     ctypes face of the C-ABI
  calibration.py, camera.py, pose_set.py, board.py, parameters.py   host mirror of the reference interface
  synthetic.py  {N_cam, N_frame, N_board, K_corners} scene generator for tests and bench.py
"""
__version__ = "0.1.0"
