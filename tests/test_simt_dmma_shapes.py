"""CPU: the host meaning of the fp64 mma helpers of csrc/kernels.cuh (dmma1688, dmma1684 and dmma_quads), i.e. what every interpreter
test of k_linearize and k_lm runs: the helpers' own text, translated by tests/simt (a host build composes each m16n8k* shape from the
interpreter's m8n8k4) and run on one interpreted warp, against numpy.  The fragments are loaded with the PTX ISA layouts the kernels
use (lane = 4 grp + tig):
  a[i] = A[grp + 8 (i & 1)][tig + 4 (i >> 1)]     b[i] = B[tig + 4 i][grp]     c[i] = C[grp + 8 (i >> 1)][2 tig + (i & 1)]
The device branch of each helper (the PTX itself) is checked on the GPU by scripts/dmma_shapes.cu and by the GPU suite.
"""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

import simt

D = C.POINTER(C.c_double)
dp = lambda a: a.ctypes.data_as(D)

HARNESS = r"""
#include "simt.h"
%s
// shape 8 / 4: one mma of that K; 12 / 28: dmma_quads over 3 / 7 quads
extern "C" void run(int shape, const double* A, const double* B, double* Cm) {
  simt::launch("dmma", dim3(1), dim3(32), 0, [&]() {
    const int l = threadIdx.x, grp = l >> 2, tig = l & 3, K = shape;
    double c[4];
    for (int i = 0; i < 4; i++) c[i] = Cm[(grp + 8 * (i >> 1)) * 8 + 2 * tig + (i & 1)];
    auto a_ = [&](int i) { return A[(grp + 8 * (i & 1)) * K + tig + 4 * (i >> 1)]; };
    auto b_ = [&](int i) { return B[(tig + 4 * i) * 8 + grp]; };
    if (shape == 8) { double a[4], b[2]; for (int i = 0; i < 4; i++) a[i] = a_(i); for (int i = 0; i < 2; i++) b[i] = b_(i); dmma1688(c, a, b); }
    if (shape == 4) { double a[2], b[1]; for (int i = 0; i < 2; i++) a[i] = a_(i); b[0] = b_(0); dmma1684(c, a, b); }
    if (shape == 12) { double a[3][2], b[3]; for (int q = 0; q < 3; q++) { a[q][0] = a_(2 * q); a[q][1] = a_(2 * q + 1); b[q] = b_(q); } dmma_quads<3>(c, a, b); }
    if (shape == 28) { double a[7][2], b[7]; for (int q = 0; q < 7; q++) { a[q][0] = a_(2 * q); a[q][1] = a_(2 * q + 1); b[q] = b_(q); } dmma_quads<7>(c, a, b); }
    for (int i = 0; i < 4; i++) Cm[(grp + 8 * (i >> 1)) * 8 + 2 * tig + (i & 1)] = c[i];
  });
}
"""


def helpers():
  """The text of the fp64 mma helpers in csrc/kernels.cuh, translated for the interpreter."""
  with open(os.path.join(simt.CSRC, "kernels.cuh")) as fh: src = fh.read()
  out = []
  for name in ("dmma884", "dmma1688", "dmma1684", "dmma_quads"):
    m = re.search(r"(template <int NQ>\s*)?__device__ __forceinline__ void " + name + r"\(", src)
    assert m, name
    body = src.index("{", m.end())
    depth, i = 0, body
    while True:
      depth += {"{": 1, "}": -1}.get(src[i], 0)
      if depth == 0: break
      i += 1
    out.append(src[m.start():i + 1])
  return simt.translate("\n".join(out))


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
  d = tmp_path_factory.mktemp("dmma")
  text = helpers()
  assert text.count("simt::dmma884(") == 1
  src, so = d / "dmma.cpp", d / "libdmma.so"
  src.write_text(HARNESS % text)
  subprocess.run(["g++", "-std=c++17", "-O1", "-fPIC", "-shared", "-w", "-I", os.path.join(simt.HERE, "shim"), "-o", str(so), str(src), "-ldl"],
                 check=True)
  L = C.CDLL(str(so))
  L.run.argtypes = [C.c_int, D, D, D]
  return L


@pytest.mark.parametrize("K", [8, 4, 12, 28])
def test_emulated_mma_matches_numpy(K, lib):
  rng = np.random.default_rng(K)
  A = np.ascontiguousarray(rng.normal(size=(16, K)))
  B = np.ascontiguousarray(rng.normal(size=(K, 8)))
  C0 = np.ascontiguousarray(rng.normal(size=(16, 8)))
  Cm = C0.copy()
  lib.run(K, dp(A), dp(B), dp(Cm))
  np.testing.assert_allclose(Cm, C0 + A @ B, rtol=1e-13, atol=1e-13)


def test_each_fragment_slot_lands_where_the_layout_says(lib):
  """A single non-zero entry of A and of B: the product has one non-zero entry, at the row of A's entry and the column of B's."""
  for K in (8, 4):
    for r, k, n in ((0, 0, 0), (9, K - 1, 7), (15, K // 2, 3), (7, 1, 5)):
      A = np.zeros((16, K)); B = np.zeros((K, 8)); Cm = np.zeros((16, 8))
      A[r, k] = 2.0; B[k, n] = 3.0
      lib.run(K, dp(A), dp(B), dp(Cm))
      expect = np.zeros((16, 8)); expect[r, n] = 6.0
      np.testing.assert_array_equal(Cm, expect)
