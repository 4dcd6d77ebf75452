"""The NumPy restatement of densification (tests/densify_oracle.py) checked on the host: the generator against a plain-integer
SplitMix64, build_rotation against its definition, and the row order on hand-made classes."""
import numpy as np

import densify_oracle as do


def test_mix64_matches_integer_restatement():
    rng = np.random.default_rng(1)
    z = rng.integers(0, 2 ** 63, 200, dtype=np.uint64) * np.uint64(2) + rng.integers(0, 2, 200, dtype=np.uint64)
    got = do.mix64(z)
    for a, b in zip(z.tolist(), got.tolist()):
        assert do.mix64_int(a) == b


def test_uniforms_follow_the_stated_counter():
    seed, call = 0xDEADBEEF12345678, 3
    rows = np.array([0, 1, 77, 2 ** 31 + 5, 2 ** 32 - 1], np.uint64)
    u1, u2 = do.uniforms(seed, call, rows)
    for i, row in enumerate(rows.tolist()):
        for a in range(3):
            k = (((call + 1) << 32) + row) * 3 + a & do.MASK
            r = do.mix64_int((seed + (k + 1) * do.GOLDEN) & do.MASK)
            assert u1[i, a] == np.float32((r >> 40) * 2.0 ** -24)
            assert u2[i, a] == np.float32(((r >> 16) & 0xFFFFFF) * 2.0 ** -24)
    assert u1.dtype == np.float32 and np.all((u1 >= 0) & (u1 < 1)) and np.all((u2 >= 0) & (u2 < 1))
    # another call or another seed draws other bits
    assert not np.array_equal(do.uniforms(seed, call + 1, rows)[0], u1)
    assert not np.array_equal(do.uniforms(seed + 1, call, rows)[0], u1)


def test_build_rotation_and_split_geometry():
    rng = np.random.default_rng(2)
    q = rng.normal(size=(500, 4))
    q = (q / np.linalg.norm(q, axis=1, keepdims=True)).astype(np.float32)
    R = do.build_rotation(q).astype(np.float64)
    eye = np.broadcast_to(np.eye(3), R.shape)
    assert np.abs(R @ np.transpose(R, (0, 2, 1)) - eye).max() < 4e-6
    assert np.all(np.abs(np.linalg.det(R) - 1) < 4e-6)
    ident = do.build_rotation(np.array([[1, 0, 0, 0]], np.float32))[0]
    assert np.array_equal(ident, np.eye(3, dtype=np.float32))
    p = rng.normal(size=(500, 3)).astype(np.float32)
    s = rng.uniform(0.01, 1, (500, 3)).astype(np.float32)
    assert np.array_equal(do.split_xyz(p, s, q, np.zeros((500, 3), np.float32)), p)
    z = rng.normal(size=(500, 3)).astype(np.float32)
    want = p.astype(np.float64) + np.einsum("nij,nj->ni", R, s.astype(np.float64) * z)
    assert np.abs(do.split_xyz(p, s, q, z) - want).max() < 1e-5


def test_classes_and_row_order():
    accum = np.array([5, 5, 1, 5, 5, 0, 5, 3], np.float32)
    denom = np.array([1, 1, 1, 1, 1, 0, 1, 2], np.float32)
    smax = np.array([1, 1, 1, 0.1, 2, 1, 0.1, 0.1], np.float32)
    # row 0 is sky; threshold 1.5: rows 1, 3, 4, 6, 7 (3/2 = 1.5) selected; clone iff smax <= 0.01 * 50 = 0.5
    cls = do.classes(accum, denom, smax, 1, 1.5, 0.01, 50.0)
    assert cls.tolist() == [0, 2, 0, 1, 2, 0, 1, 1]
    src, n = do.select(cls)
    assert n == dict(kept=6, cloned=3, split=2, total=13)
    assert src.tolist() == [0, 2, 3, 5, 6, 7, 3, 6, 7, 1, 4, 1, 4]
    # just above the exact 3/2: row 7 leaves the selection
    assert do.classes(accum, denom, smax, 1, np.nextafter(np.float32(1.5), np.float32(2)), 0.01, 50.0)[7] == 0
