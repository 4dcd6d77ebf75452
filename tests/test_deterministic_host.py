"""The deterministic render backward's documented association, restated on the host (deterministic_oracle.py), and the size
of its workspace (glic_deterministic_bytes).  No GPU needed."""
import numpy as np
import pytest

from deterministic_oracle import fold, fold_entries, scatter


def _left_fold(v):
    s = np.float32(v[0])
    for x in v[1:]:
        s = np.float32(s + np.float32(x))
    return s


def test_order_changes_the_result_and_the_fold_keeps_it():
    """[1e8, 1, -1e8] gives 0 left to right and 1 once the large terms cancel first: the fold is the left-to-right one"""
    v = np.array([1e8, 1.0, -1e8], np.float32)
    assert fold(v) == np.float32(0.0)
    assert fold(v[[0, 2, 1]]) == np.float32(1.0)


@pytest.mark.parametrize("n", [1, 31, 32, 33, 1025])
def test_fold_is_chunked_left_fold(n):
    rng = np.random.default_rng(n)
    v = (rng.normal(size=n) * 10.0 ** rng.integers(-4, 5, size=n)).astype(np.float32)
    chunks = [_left_fold(v[c:c + 32]) for c in range(0, n, 32)]
    want = _left_fold(np.array(chunks, np.float32))
    assert fold(v).tobytes() == want.tobytes()
    if n <= 32:
        assert fold(v).tobytes() == _left_fold(v).tobytes()


def test_fold_of_a_long_run_differs_from_the_strict_left_fold_where_it_should():
    """33 entries: the 33rd is added to the sum of the first 32, which is the strict left fold as well; from 64 + 1 entries on,
    the chunk sums are folded separately"""
    v = np.array([1e8] + [1.0] * 31 + [-1e8] + [1.0] * 31 + [0.5], np.float32)
    chunks = [_left_fold(v[:32]), _left_fold(v[32:64]), _left_fold(v[64:])]
    assert fold(v) == _left_fold(np.array(chunks, np.float32))
    assert fold(v) != _left_fold(v)


def test_fold_entries_matches_fold_per_gid():
    rng = np.random.default_rng(3)
    lens = [1, 31, 32, 33, 1025, 2, 64, 65]
    gid = np.repeat(np.arange(len(lens)) * 7 + 1, lens)
    vals = (rng.normal(size=(gid.size, 9)) * 10.0 ** rng.integers(-3, 4, size=(gid.size, 9))).astype(np.float32)
    gids, sums, counts, abs_sums = fold_entries(gid, vals)
    assert list(counts) == lens
    start = 0
    for i, n in enumerate(lens):
        assert gids[i] == gid[start]
        assert sums[i].tobytes() == fold(vals[start:start + n]).tobytes()
        np.testing.assert_allclose(abs_sums[i], np.abs(vals[start:start + n].astype(np.float64)).sum(0))
        start += n
    out = scatter(gids.max() + 1, gids, sums)
    assert out["dL_dopacity"][gids[3], 0] == sums[3, 8]
    assert out["dL_dconic"][gids[4], 3] == sums[4, 4] and out["dL_dconic"][gids[4], 2] == 0
    assert not out["dL_dcolors"][0].any()


def test_fold_entries_empty():
    gids, sums, counts, _ = fold_entries(np.zeros(0, np.int64), np.zeros((0, 9), np.float32))
    assert gids.size == 0 and sums.shape == (0, 9) and counts.size == 0


def test_deterministic_bytes_covers_the_carve_and_grows():
    from gaussian_lic_b200 import capi
    lib = capi.lib
    for R, W, H in [(1, 16, 16), (100000, 320, 208), (4 << 20, 1920, 1080)]:
        b = lib.glic_deterministic_bytes(R, W, H)
        n = 32 * lib.glic_max_buckets(R, W, H)
        # count | keys[2] | idx[2] | vals[9] | sort temp, each 128-byte aligned
        assert b >= n * (4 * 4 + 36) + lib.glic_sort_temp_bytes(n)
        assert b <= n * (4 * 4 + 36) + lib.glic_sort_temp_bytes(n) + 8 * 128
        assert lib.glic_deterministic_bytes(2 * R, W, H) >= b
        if R > 1:
            assert lib.glic_deterministic_bytes(2 * R, W, H) > b
        assert lib.glic_deterministic_bytes(R, 2 * W, 2 * H) >= b
    assert lib.glic_deterministic_bytes(1000, 1920, 1080) > lib.glic_deterministic_bytes(1000, 320, 208)
    assert lib.glic_deterministic_bytes(0, 320, 208) > 0
