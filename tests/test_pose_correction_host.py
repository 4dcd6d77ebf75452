"""glic_pose_correction_record and glic_sh_rotation on the host (no GPU): the record's R, t and q against the NumPy restatement
bit for bit, and the SH band matrices against their definition, orthogonality, composition and an independent fit."""
import numpy as np
import pytest

from gaussian_lic_b200 import capi
from gaussian_lic_b200.mapper import pose_correction_record, sh_rotation
import pose_correction_oracle as O


def _rot(axis, angle):
    a = np.asarray(axis, np.float64)
    a = a / np.linalg.norm(a)
    K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    return np.eye(3) + np.sin(angle) * K + (1 - np.cos(angle)) * K @ K


def _random_pose(rng):
    return _rot(rng.normal(size=3), rng.uniform(0, np.pi)).astype(np.float32), rng.normal(scale=5, size=3).astype(np.float32)


CASES = [
    ("identity", np.eye(3), np.eye(3)),
    ("180 about x", np.eye(3), _rot([1, 0, 0], np.pi)),
    ("180 about y", np.eye(3), _rot([0, 1, 0], np.pi)),
    ("180 about z", np.eye(3), _rot([0, 0, 1], np.pi)),
    ("180 tilted, r = 0 tie to a negative lead", np.eye(3), 2 * np.outer([-1, 2, 0], [-1, 2, 0]) / 5 - np.eye(3)),
    ("180 about (1, -1, 0)", np.eye(3), 2 * np.outer([1, -1, 0], [1, -1, 0]) / 2 - np.eye(3)),
    ("near 180", _rot([0.3, -1, 2], 0.4), _rot([1, 2, 3], np.pi - 1e-6) @ _rot([0.3, -1, 2], 0.4)),
    ("near 180 about z", np.eye(3), _rot([1e-4, 0, 1], np.pi - 1e-7)),
    ("small", _rot([1, 1, 0], 0.7), _rot([2, -1, 1], 1e-6) @ _rot([1, 1, 0], 0.7)),
]


@pytest.mark.parametrize("name,R_old,R_new", CASES, ids=[c[0] for c in CASES])
def test_record_matches_the_restatement_bit_for_bit(name, R_old, R_new):
    rng = np.random.default_rng(len(name))
    t_old, t_new = rng.normal(size=3).astype(np.float32), rng.normal(size=3).astype(np.float32)
    Ro, Rn = np.asarray(R_old, np.float32), np.asarray(R_new, np.float32)
    r = pose_correction_record(Ro, t_old, Rn, t_new, 3)
    R, t = O.record_rt(Ro, t_old, Rn, t_new)
    q = O.record_q(R)
    assert np.array_equal(r["R"].reshape(9), R) and np.array_equal(r["t"], t)
    assert np.array_equal(r["q"], q) and np.signbit(r["q"]).tolist() == np.signbit(q).tolist(), (r["q"], q)
    assert r["q"][0] >= 0 and abs(np.linalg.norm(r["q"]) - 1) < 1e-15
    # q is the rotation of dR to the float precision of the poses
    assert np.abs(O.quat_matrix(r["q"]) - R.reshape(3, 3)).max() < 1e-6
    # its band matrices are glic_sh_rotation's of q
    assert all(np.array_equal(a, b) for a, b in zip(r["sh"], sh_rotation(r["q"], 3)))


def test_r_zero_tie_rule():
    n = np.array([-1, 2, 0]) / np.sqrt(5)
    r = pose_correction_record(np.eye(3), np.zeros(3), (2 * np.outer(n, n) - np.eye(3)).astype(np.float32), np.zeros(3), 1)
    q = r["q"]
    assert q[0] == 0 and not np.signbit(q[0]) and q[1] > 0 and q[2] < 0 and q[3] == 0, q


def test_random_records_match_the_restatement():
    rng = np.random.default_rng(1)
    for _ in range(200):
        (Ro, to), (Rn, tn) = _random_pose(rng), _random_pose(rng)
        r = pose_correction_record(Ro, to, Rn, tn, 0)
        R, t = O.record_rt(Ro, to, Rn, tn)
        assert np.array_equal(r["R"].reshape(9), R) and np.array_equal(r["t"], t) and np.array_equal(r["q"], O.record_q(R))
        assert r["sh"] == []                             # degree 0: no band matrix


def _unit_quats(rng, n):
    q = rng.normal(size=(n, 4))
    return q / np.linalg.norm(q, axis=1, keepdims=True)


def test_band_matrices_satisfy_their_definition():
    rng = np.random.default_rng(2)
    d = rng.normal(size=(1000, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    for q in list(_unit_quats(rng, 20)) + [np.array([1.0, 0, 0, 0]), np.array([0.0, 0, 0, 1])]:
        A = sh_rotation(q, 3)
        Rt_d = d @ O.quat_matrix(q)                      # R(q)^T d
        for l in range(1, 4):
            c = rng.normal(size=2 * l + 1)
            lhs = O.band_basis(l, d) @ (A[l - 1] @ c)
            rhs = O.band_basis(l, Rt_d) @ c
            assert np.abs(lhs - rhs).max() < 1e-12, (l, np.abs(lhs - rhs).max())
            assert np.abs(A[l - 1] @ A[l - 1].T - np.eye(2 * l + 1)).max() < 1e-12


def test_band_matrices_compose_and_match_an_independent_fit():
    rng = np.random.default_rng(3)
    for q1, q2 in zip(_unit_quats(rng, 10), _unit_quats(rng, 10)):
        q12 = O.quat_mul(q1, q2)
        q12 /= np.linalg.norm(q12)
        A1, A2, A12 = sh_rotation(q1), sh_rotation(q2), sh_rotation(q12)
        for l in range(3):
            assert np.abs(A12[l] - A1[l] @ A2[l]).max() < 1e-12
        for a, f in zip(A12, O.sh_fit(q12, 3)):
            assert np.abs(a - f).max() < 1e-10


def test_identity_is_the_identity():
    r = pose_correction_record(np.eye(3), np.ones(3), np.eye(3), np.ones(3), 3)
    assert np.array_equal(r["q"], [1, 0, 0, 0]) and not np.any(r["t"])
    for l, A in enumerate(r["sh"], 1):
        assert np.abs(A - np.eye(2 * l + 1)).max() < 1e-14


def test_bands_above_the_degree_are_zero():
    import ctypes as C
    out = capi.RigidCorrection()
    R = (C.c_float * 9)(*_rot([1, 2, 3], 0.7).astype(np.float32).reshape(9))
    t = (C.c_float * 3)(1.0, 2.0, 3.0)
    I9 = (C.c_float * 9)(*np.eye(3, dtype=np.float32).reshape(9))
    for degree in range(4):
        assert capi.lib.glic_pose_correction_record(I9, t, R, t, degree, C.byref(out)) == 0
        n = {0: 0, 1: 9, 2: 34, 3: 83}[degree]
        assert all(v != 0 for v in out.sh[:3]) == (degree > 0) and not any(out.sh[n:]), degree


def test_bad_arguments_are_refused():
    out = capi.RigidCorrection()
    import ctypes as C
    I9 = (C.c_float * 9)(*np.eye(3, dtype=np.float32).reshape(9))
    z3 = (C.c_float * 3)()
    assert capi.lib.glic_pose_correction_record(I9, z3, I9, z3, 4, C.byref(out)) != 0
    assert capi.lib.glic_pose_correction_record(None, z3, I9, z3, 3, C.byref(out)) != 0
    assert capi.lib.glic_sh_rotation(None, 3, (C.c_double * 83)()) != 0
