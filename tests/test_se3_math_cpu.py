"""malio_se3.h without a GPU: the library's one source of quaternion and SE(3) algebra, compiled by g++ with the Makefile's host
flags into a small shim, against float64 restatements of Eigen's and quat_ops.h's expressions in their operation order.

Python floats are IEEE doubles and every operation rounds once (no FMA), so the shim and the restatement agree bit for bit,
signed zeros included: q_rot, q_rot_conj, q_mul, q_to_R, q_yaw_mul (against reloc_ref.candidate_rotations, whose math.cos /
math.sin are the C library's the header calls), mul3, mul4, inv_se3, and quat_from_R on each of its four branches.  Inputs are
non-unit quaternions, vectors and matrices over magnitudes from 1e-6 to 1e6, plus zeros and signed zeros.  log_so3, exp_se3
and log_se3 call acos / sin / tan, where the C library and Python need not agree in the last ulp: the spline tests cover them
within a tolerance."""
import ctypes as C
import math
import os
import re
import subprocess

import numpy as np
import pytest

import reloc_ref as RR

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "ma-lio_b200", "csrc")

SHIM = r"""
#include "malio_se3.h"
using namespace malio_se3;
extern "C" {
void t_q_rot(const double* q, const double* v, double* o, int n) { for (int i = 0; i < n; ++i) q_rot(q + 4 * i, v + 3 * i, o + 3 * i); }
void t_q_rot_conj(const double* q, const double* v, double* o, int n) { for (int i = 0; i < n; ++i) q_rot_conj(q + 4 * i, v + 3 * i, o + 3 * i); }
void t_q_mul(const double* a, const double* b, double* o, int n) { for (int i = 0; i < n; ++i) q_mul(a + 4 * i, b + 4 * i, o + 4 * i); }
void t_q_to_R(const double* q, double* R, int n) { for (int i = 0; i < n; ++i) q_to_R(q + 4 * i, R + 9 * i); }
void t_q_yaw_mul(const double* theta, const double* q, double* o, int n) { for (int i = 0; i < n; ++i) q_yaw_mul(theta[i], q + 4 * i, o + 4 * i); }
void t_mul3(const double* A, const double* B, double* C, int n) { for (int i = 0; i < n; ++i) mul3(A + 9 * i, B + 9 * i, C + 9 * i); }
void t_mul4(const double* A, const double* B, double* C, int n) { for (int i = 0; i < n; ++i) mul4(A + 16 * i, B + 16 * i, C + 16 * i); }
void t_inv_se3(const double* T, double* Ti, int n) { for (int i = 0; i < n; ++i) inv_se3(T + 16 * i, Ti + 16 * i); }
void t_quat_from_R(const double* m, double* q, int n) { for (int i = 0; i < n; ++i) quat_from_R(m + 9 * i, q + 4 * i); }
}
"""


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    mk = open(os.path.join(CSRC, "Makefile")).read()
    flags = [f for f in re.search(r"^CXXFLAGS := (.*)$", mk, re.M).group(1).split() if f != "$(INC)"]
    d = tmp_path_factory.mktemp("se3_math")
    (d / "shim.cpp").write_text(SHIM)
    so = d / "libse3shim.so"
    subprocess.run(["/usr/bin/g++", *flags, "-I" + os.path.join(ROOT, "include"), "-I" + CSRC, "-shared", str(d / "shim.cpp"),
                    "-o", str(so)], check=True)
    return C.CDLL(str(so))


def call(lib, name, out_width, *args):
    """t_<name> over the rows of the input arrays -> (rows, out_width)"""
    args = [np.ascontiguousarray(a, np.float64) for a in args]
    o = np.zeros((args[0].shape[0], out_width))
    getattr(lib, "t_" + name)(*[a.ctypes.data_as(C.c_void_p) for a in args], o.ctypes.data_as(C.c_void_p), C.c_int(o.shape[0]))
    return o


def assert_bits(got, want):
    want = np.asarray(want, np.float64).reshape(got.shape)
    bad = np.nonzero(got.view(np.uint64) != want.view(np.uint64))
    assert bad[0].size == 0, f"{bad[0].size} differing values, first at {bad[0][0]}: {got[bad][0]!r} != {want[bad][0]!r}"


def rows(rng, n, width):
    """n random rows at magnitudes 1e-6 .. 1e6, then 128 rows of 0.0, -0.0, 1.0 and -2.5, the first two all 0.0 and all -0.0"""
    r = rng.standard_normal((n, width)) * 10.0 ** rng.integers(-6, 7, (n, 1))
    special = rng.choice(np.array([0.0, -0.0, 1.0, -2.5]), (128, width))
    special[0], special[1] = 0.0, -0.0
    return np.vstack([r, special])


# ---------------------------------------------------------------- restatements (Eigen's operation order)
def cross(a, b):
    return [a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]]


def q_rot(q, v):   # Quaternion::_transformVector: uv = q.vec() x v; uv += uv; v + q.w() * uv + q.vec() x uv
    qv = q[1:4]
    uv = cross(qv, v)
    uv = [u + u for u in uv]
    c = cross(qv, uv)
    return [v[i] + q[0] * uv[i] + c[i] for i in range(3)]


def q_mul(a, b):   # quat_product
    return [a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3], a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2],
            a[0] * b[2] + a[2] * b[0] + a[3] * b[1] - a[1] * b[3], a[0] * b[3] + a[3] * b[0] + a[1] * b[2] - a[2] * b[1]]


def q_to_R(q):   # QuaternionBase::toRotationMatrix
    w, x, y, z = q
    tx, ty, tz = 2 * x, 2 * y, 2 * z
    twx, twy, twz, txx, txy, txz, tyy, tyz, tzz = tx * w, ty * w, tz * w, tx * x, ty * x, tz * x, ty * y, tz * y, tz * z
    return [1 - (tyy + tzz), txy - twz, txz + twy, txy + twz, 1 - (txx + tzz), tyz - twx, txz - twy, tyz + twx, 1 - (txx + tyy)]


def matmul(A, B, n):   # row-major n x n, k ascending
    out = []
    for i in range(n):
        for j in range(n):
            s = A[n * i] * B[j]
            for k in range(1, n):
                s = s + A[n * i + k] * B[n * k + j]
            out.append(s)
    return out


def inv_se3(T):   # quat_ops.h Inv: [R^T, -R^T p; 0 0 0 1]
    Ti = [0.0] * 16
    for i in range(3):
        for j in range(3):
            Ti[4 * i + j] = T[4 * j + i]
        Ti[4 * i + 3] = -(Ti[4 * i] * T[3] + Ti[4 * i + 1] * T[7] + Ti[4 * i + 2] * T[11])
    Ti[15] = 1.0
    return Ti


def quat_from_R(m):   # Eigen 3.3 quaternionbase_assign_impl<Matrix3>
    t = m[0] + m[4] + m[8]
    if t > 0.0:
        t = math.sqrt(t + 1.0)
        w = 0.5 * t
        t = 0.5 / t
        return [w, (m[7] - m[5]) * t, (m[2] - m[6]) * t, (m[3] - m[1]) * t], 3
    i = 0
    if m[4] > m[0]:
        i = 1
    if m[8] > m[4 * i]:
        i = 2
    j, k = (i + 1) % 3, (i + 2) % 3
    t = math.sqrt(m[4 * i] - m[4 * j] - m[4 * k] + 1.0)
    qv = [0.0] * 3
    qv[i] = 0.5 * t
    t = 0.5 / t
    w = (m[3 * k + j] - m[3 * j + k]) * t
    qv[j] = (m[3 * j + i] + m[3 * i + j]) * t
    qv[k] = (m[3 * k + i] + m[3 * i + k]) * t
    return [w] + qv, i


def conj(q):
    return [q[0], -q[1], -q[2], -q[3]]


# ---------------------------------------------------------------- tests
def test_quaternion_vector_products(shim):
    rng = np.random.default_rng(71)
    q, v, b = rows(rng, 3000, 4), rows(rng, 3000, 3), rows(rng, 3000, 4)
    assert_bits(call(shim, "q_rot", 3, q, v), [q_rot(list(x), list(y)) for x, y in zip(q, v)])
    assert_bits(call(shim, "q_rot_conj", 3, q, v), [q_rot(conj(list(x)), list(y)) for x, y in zip(q, v)])
    assert_bits(call(shim, "q_mul", 4, q, b), [q_mul(list(x), list(y)) for x, y in zip(q, b)])
    assert_bits(call(shim, "q_to_R", 9, q), [q_to_R(list(x)) for x in q])


def test_yaw_product_is_the_relocalization_candidates(shim):
    rng = np.random.default_rng(72)
    for rot, yaw_lo, yaw_step, n_yaw in [(rows(rng, 1, 4)[0], -math.pi, 2 * math.pi / 360, 361),
                                         (rows(rng, 1, 4)[0], -0.3, 0.01, 61),
                                         ([1.0, 0.0, -0.0, 0.0], -1e3, 7.3, 300),
                                         ([0.0, -0.0, 0.0, -0.0], 0.0, 1e-9, 5)]:
        theta = [yaw_lo + float(k) * yaw_step for k in range(n_yaw)]   # malio_relocalize's theta_k
        got = call(shim, "q_yaw_mul", 4, theta, np.tile(np.asarray(rot, np.float64), (n_yaw, 1)))
        assert_bits(got, RR.candidate_rotations(rot, yaw_lo, yaw_step, n_yaw))


def test_matrix_products_and_rigid_inverse(shim):
    rng = np.random.default_rng(73)
    A, B = rows(rng, 2000, 9), rows(rng, 2000, 9)
    assert_bits(call(shim, "mul3", 9, A, B), [matmul(list(x), list(y), 3) for x, y in zip(A, B)])
    T, U = rows(rng, 2000, 16), rows(rng, 2000, 16)
    T[:, 12:] = U[:, 12:] = [0.0, 0.0, 0.0, 1.0]      # homogeneous, as the callers pass them
    assert_bits(call(shim, "mul4", 16, T, U), [matmul(list(x), list(y), 4) for x, y in zip(T, U)])
    assert_bits(call(shim, "inv_se3", 16, T), [inv_se3(list(x)) for x in T])


def test_quaternion_from_matrix_every_branch(shim):
    rng = np.random.default_rng(74)
    # rotation matrices of random unit quaternions, general matrices, and matrices near the identity (trace > 0) and near the
    # half-turns about x, y and z (i = 0, 1, 2), perturbed at magnitudes 1e-8 .. 1e-1
    M = [q_to_R(list(x / np.linalg.norm(x))) for x in rng.standard_normal((800, 4))] + list(rows(rng, 800, 9))
    for diag in [(1, 1, 1), (1, -1, -1), (-1, 1, -1), (-1, -1, 1)]:
        for e in 10.0 ** np.arange(-8, 0):
            M += list(np.diag(diag).ravel() + e * rng.standard_normal((50, 9)))
    want, branch = zip(*[quat_from_R(list(m)) for m in M])
    counts = np.bincount(branch, minlength=4)
    assert counts.min() >= 200, counts               # [i = 0, i = 1, i = 2, trace > 0]
    assert_bits(call(shim, "quat_from_R", 4, M), want)
