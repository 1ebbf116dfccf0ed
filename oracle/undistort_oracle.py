"""numpy restatement of what the reference does with OpenCV to remap an image through a finished calibration's map (camera.py:244-258):
cv2.remap(image, map, None, INTER_CUBIC) with the default constant-zero border, for uint8 images, and OpenCV's sensor tilt matrix.  The
map itself (R = I and newK = K for the undistortion) is restated in oracle/rectify_oracle.py.

This is the arithmetic the device kernels in multical_b200/csrc/undistort_kernels.cuh follow; the tests compare both this and the
device against live cv2.
"""
import numpy as np

TAB = 32                  # INTER_TAB_SIZE: 1/32-pixel sub-positions
COEF_BITS = 15            # INTER_REMAP_COEF_BITS
COEF_SCALE = 1 << COEF_BITS


def cubic_coeffs(x):
  """The four 1-D cubic weights at sub-position x (float32 arithmetic, A = -0.75)."""
  f = np.float32
  A, x = f(-0.75), f(x)
  one = f(1)
  c0 = ((A * (x + one) - f(5) * A) * (x + one) + f(8) * A) * (x + one) - f(4) * A
  c1 = ((A + f(2)) * x - (A + f(3))) * x * x + one
  y = one - x
  c2 = ((A + f(2)) * y - (A + f(3))) * y * y + one
  c3 = one - c0 - c1 - c2
  return np.array([c0, c1, c2, c3], np.float32)


def cubic_table():
  """int32 [32*32][16]: entry (Y&31)*32 + (X&31) holds the 4x4 fixed-point weights (row-major, rows = y taps)."""
  one_d = [cubic_coeffs(np.float32(k) * np.float32(1.0 / TAB)) for k in range(TAB)]
  tab = np.zeros((TAB * TAB, 16), np.int32)
  for i in range(TAB):
    for j in range(TAB):
      w = np.outer(one_d[i], one_d[j]).astype(np.float32)            # float32 products
      t = np.rint(w * np.float32(COEF_SCALE)).astype(np.int32).reshape(4, 4)
      diff = int(t.sum()) - COEF_SCALE
      if diff:
        mk = Mk = (2, 2)
        for k1 in (2, 3):
          for k2 in (2, 3):
            if t[k1, k2] < t[mk]: mk = (k1, k2)
            elif t[k1, k2] > t[Mk]: Mk = (k1, k2)
        if diff < 0: t[Mk] -= diff
        else: t[mk] -= diff
      tab[i * TAB + j] = t.reshape(16)
  return tab


def fixed_point_map(m):
  """float32 [h][w][2] map -> (sx, sy, table index) as remap reads it: X = rint(32 x), taps from (X >> 5) - 1."""
  m = np.asarray(m, np.float32)

  def cv_round(v):                      # ties to even; NaN and values outside int32 give INT_MIN, as OpenCV's x86 conversion does
    ok = (v >= -2.0 ** 31) & (v < 2.0 ** 31)
    return np.where(ok, np.rint(np.where(ok, v, 0)), -2.0 ** 31).astype(np.int64)

  with np.errstate(invalid="ignore", over="ignore"):
    X = cv_round(m[..., 0] * np.float32(TAB))
    Y = cv_round(m[..., 1] * np.float32(TAB))
  sx = np.clip(X >> 5, -32768, 32767) - 1
  sy = np.clip(Y >> 5, -32768, 32767) - 1
  return sx, sy, (Y & 31) * TAB + (X & 31)


def remap_cubic(src, m):
  """cv2.remap(src, m, None, INTER_CUBIC) for uint8 src [h][w] or [h][w][3] and a float32 map [H][W][2]."""
  src = np.asarray(src)
  gray = src.ndim == 2
  s = src[..., None] if gray else src
  h, w, cn = s.shape
  sx, sy, idx = fixed_point_map(m)
  tab = cubic_table()[idx]                                            # [H][W][16]
  acc = np.zeros(sx.shape + (cn,), np.int64)
  for ky in range(4):
    yy = sy + ky
    for kx in range(4):
      xx = sx + kx
      inside = (xx >= 0) & (xx < w) & (yy >= 0) & (yy < h)
      v = s[np.clip(yy, 0, h - 1), np.clip(xx, 0, w - 1)].astype(np.int64)
      acc += np.where(inside[..., None], v, 0) * tab[..., 4 * ky + kx, None]
  out = np.clip((acc + (1 << (COEF_BITS - 1))) >> COEF_BITS, 0, 255).astype(np.uint8)
  return out[..., 0] if gray else out


def _tilt(tx, ty):
  cx, sx, cy, sy = np.cos(tx), np.sin(tx), np.cos(ty), np.sin(ty)
  Rx = np.array([[1, 0, 0], [0, cx, sx], [0, -sx, cx]])
  Ry = np.array([[cy, 0, -sy], [0, 1, 0], [sy, 0, cy]])
  R = Ry @ Rx
  Pz = np.array([[R[2, 2], 0, -R[0, 2]], [0, R[2, 2], -R[1, 2]], [0, 0, 1]])
  return Pz @ R
