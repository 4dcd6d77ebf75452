"""The onesweep radix sort pass by pass against numpy's stable argsort, bit for bit: the 32-bit-key sort of the binning
(depth keys, tile ids; capacity-sized launches that read the true count from the device), the 64-bit sort, tile sizes
and counts around the small/big tile switch, degenerate digit distributions, the tile sort as the forward runs it (digit
histograms built by the key emission) at 13 and 16 tile bits, and run-to-run determinism."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

NUM_SMS = 132
SORT_SMALL_LIMIT = NUM_SMS * 4 * 256 * 16          # radix_sort.cu: below this many pairs the 1024-pair tile is used


def _sort_u32(keys, vals, end_bit, n_launch=None, n_true=None):
    """glic_debug_sort_pairs_u32 on n_launch pairs (default: all), of which only the first n_true (read from the device)
    are live -> (keys, vals) of the live prefix, sorted."""
    from gaussian_lic_b200 import capi
    lib = capi.lib
    n = len(keys) if n_launch is None else n_launch
    dev = torch.device("cuda:0")
    k = [torch.as_tensor(keys.view(np.int32)).to(dev), torch.empty(n, dtype=torch.int32, device=dev)]
    v = [torch.as_tensor(vals.view(np.int32)).to(dev), torch.empty(n, dtype=torch.int32, device=dev)]
    temp = torch.empty(lib.glic_sort_temp_bytes(n), dtype=torch.uint8, device=dev)
    n_dev = None if n_true is None else torch.tensor([n_true], dtype=torch.int32, device=dev)
    cur = lib.glic_debug_sort_pairs_u32(n, end_bit, capi.ptr(k[0]), capi.ptr(v[0]), capi.ptr(k[1]), capi.ptr(v[1]),
                                        None if n_dev is None else capi.ptr(n_dev), capi.ptr(temp), temp.numel(), None)
    assert cur in (0, 1), cur
    torch.cuda.synchronize()
    live = n if n_true is None else n_true
    return k[cur][:live].cpu().numpy().view(np.uint32), v[cur][:live].cpu().numpy().view(np.uint32)


def _expect(keys, vals, end_bit):
    order = np.argsort(keys & np.uint32((1 << end_bit) - 1) if end_bit < 32 else keys, kind="stable")
    return keys[order], vals[order]


def _check_u32(keys, vals, end_bit, **kw):
    ko, vo = _sort_u32(keys, vals, end_bit, **kw)
    live = kw.get("n_true") or len(keys)
    ke, ve = _expect(keys[:live], vals[:live], end_bit)
    np.testing.assert_array_equal(ko, ke)
    np.testing.assert_array_equal(vo, ve)


def _rng(seed):
    return np.random.Generator(np.random.Philox(seed))


SIZES = [1, 1000, 4097, 100_003, SORT_SMALL_LIMIT - 1, SORT_SMALL_LIMIT + 1]


@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("end_bit", [13, 16, 32])
def test_u32_random_keys(n, end_bit):
    rng = _rng(n + end_bit)
    keys = rng.integers(0, 1 << end_bit, n, dtype=np.uint64).astype(np.uint32)
    vals = rng.permutation(n).astype(np.uint32)
    _check_u32(keys, vals, end_bit)


def test_u32_depth_keys_float_bits():
    """the depth sort's keys: float bits of positive depths, with exact ties"""
    rng = _rng(3)
    depth = rng.uniform(0.2, 100.0, 500_000).astype(np.float32)
    depth[::7] = depth[3]
    keys = depth.view(np.uint32)
    _check_u32(keys, np.arange(len(keys), dtype=np.uint32), 32)


@pytest.mark.parametrize("end_bit", [13, 16, 32])
@pytest.mark.parametrize("kind", ["all_equal", "one_digit", "every_digit"])
@pytest.mark.parametrize("n", [4097, SORT_SMALL_LIMIT + 1])
def test_u32_digit_distributions(end_bit, kind, n):
    rng = _rng(n + end_bit)
    if kind == "all_equal":
        keys = np.full(n, (1 << end_bit) - 1 if end_bit < 32 else 0xDEADBEEF, np.uint32)
    elif kind == "one_digit":                       # the lowest pass sees one digit, the others many
        keys = (rng.integers(0, 1 << (end_bit - 8), n, dtype=np.uint64) << np.uint64(8) | np.uint64(0x5A)).astype(np.uint32)
    else:                                           # every digit of every pass occurs, in a shuffled order
        keys = (rng.permutation(n).astype(np.uint64) % np.uint64(1 << end_bit)).astype(np.uint32)
    _check_u32(keys, np.arange(n, dtype=np.uint32), end_bit)


@pytest.mark.parametrize("n_launch,n_true", [(5000, 1), (5000, 4096), (SORT_SMALL_LIMIT + 5000, 1_000_003),
                                             (SORT_SMALL_LIMIT + 5000, SORT_SMALL_LIMIT + 4999)])
@pytest.mark.parametrize("end_bit", [13, 16])
def test_u32_device_count_below_launch(n_launch, n_true, end_bit):
    """capacity-sized launch, true count on the device: the pairs past it are neither read nor written"""
    rng = _rng(n_true)
    keys = rng.integers(0, 1 << end_bit, n_launch, dtype=np.uint64).astype(np.uint32)
    vals = np.arange(n_launch, dtype=np.uint32)
    _check_u32(keys, vals, end_bit, n_launch=n_launch, n_true=n_true)


@pytest.mark.parametrize("n", [1, 4097, SORT_SMALL_LIMIT - 1, SORT_SMALL_LIMIT + 1])
def test_u64_45_bit_keys(n):
    from gaussian_lic_b200 import ops, synthetic as syn
    keys, vals = syn.make_sort_pairs(n, seed=n)
    ko, vo = ops.sort_pairs(torch.as_tensor(keys.view(np.int64)).cuda(), torch.as_tensor(vals.view(np.int32)).cuda(), 45)
    torch.cuda.synchronize()
    order = np.argsort(keys & np.uint64((1 << 45) - 1), kind="stable")
    np.testing.assert_array_equal(ko.cpu().numpy().view(np.uint64), keys[order])
    np.testing.assert_array_equal(vo.cpu().numpy().view(np.uint32), vals[order])


def test_two_runs_identical():
    rng = _rng(11)
    n = SORT_SMALL_LIMIT + 12345
    keys = rng.integers(0, 1 << 13, n, dtype=np.uint64).astype(np.uint32)
    vals = np.arange(n, dtype=np.uint32)
    a = _sort_u32(keys, vals, 13)
    b = _sort_u32(keys, vals, 13)
    np.testing.assert_array_equal(a[0], b[0])
    np.testing.assert_array_equal(a[1], b[1])


@pytest.mark.parametrize("W,H,bits", [(1920, 1080, 13), (4096, 4096, 16)])
def test_forward_tile_sort(W, H, bits):
    """The tile sort as the forward runs it (histograms from the key emission, capacity-sized launch, device count): the
    pair list must be every (tile, Gaussian) pair once, ordered by tile, then depth, then Gaussian index."""
    from gaussian_lic_b200 import ops, synthetic as syn
    g, cam = syn.make_frame_scene(W, H, P=20000)
    r = ops.CRasterizer(W, H, "cuda:0")
    gd = ops.scene_to_device(g)
    view = r.make_view(cam)
    runs = []
    for _ in range(2):
        r.forward(gd, view)
        d = r.debug_state()
        runs.append((d["keys_sorted"].cpu().numpy().view(np.uint64), d["point_list"].cpu().numpy().view(np.uint32)))
    T = ((W + 15) // 16) * ((H + 15) // 16)
    assert (T - 1).bit_length() == bits
    keys, pl = runs[0]
    assert r.R > 0 and len(pl) == r.R
    tile = keys >> np.uint64(32)
    depth = keys & np.uint64(0xFFFFFFFF)
    assert int(tile.max()) < T
    np.testing.assert_array_equal(np.lexsort((pl, depth, tile)), np.arange(r.R))
    tiles_touched = d["tiles_touched"].cpu().numpy()
    np.testing.assert_array_equal(np.bincount(pl, minlength=len(tiles_touched)), tiles_touched)
    assert np.unique(tile * np.uint64(len(tiles_touched)) + pl.astype(np.uint64)).size == r.R
    np.testing.assert_array_equal(runs[1][0], keys)
    np.testing.assert_array_equal(runs[1][1], pl)
