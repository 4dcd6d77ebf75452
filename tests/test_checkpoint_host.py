"""glic_mapper_checkpoint_config against a restatement of the documented checkpoint header (tests/checkpoint_format.py): it
returns the written configuration exactly and refuses malformed headers.  Host only, no GPU."""
import ctypes as C

import numpy as np
import pytest

import checkpoint_format as F

CFG = dict(width=320, height=208, fx=250.25, fy=249.75, cx=160.0, cy=104.5, sh_degree=3, position_lr=1.6e-4, feature_lr=2.5e-3,
           opacity_lr=0.05, scaling_lr=0.005, rotation_lr=0.001, lambda_dssim=0.2, scaling_scale=1.0, capacity=4096, max_iters=100,
           seed=(1 << 63) + 12345, rank=1, world=2, views_per_rank=3)


def _config(path):
    from gaussian_lic_b200 import capi
    cfg = capi.MapperConfig()
    rc = capi.lib.glic_mapper_checkpoint_config(str(path).encode(), C.byref(cfg))
    return rc, cfg


def _write(tmp_path, data, name="c.ckpt"):
    p = tmp_path / name
    p.write_bytes(data)
    return p


def test_header_round_trips_every_field(tmp_path):
    rc, cfg = _config(_write(tmp_path, F.header(CFG) + F.END))
    assert rc == 0
    for k, code in F.CONFIG_FIELDS:
        got = getattr(cfg, k)
        want = CFG[k]
        if code == "f":
            assert np.float32(got).view(np.uint32) == np.float32(want).view(np.uint32), k
        else:
            assert got == want, k
    # the header alone is enough (the sections are load_checkpoint's to check)
    rc, _ = _config(_write(tmp_path, F.header(CFG), "header_only.ckpt"))
    assert rc == 0


def test_bad_magic_and_version_are_refused(tmp_path):
    assert _config(_write(tmp_path, F.header(CFG, magic=b"GLICCKPU") + F.END))[0] == -1
    for v in (0, 2, 0xFFFFFFFF):
        assert _config(_write(tmp_path, F.header(CFG, version=v) + F.END))[0] == -1, v


def test_header_cut_at_every_byte_is_refused(tmp_path):
    h = F.header(CFG)
    assert len(h) == F.HEADER_BYTES
    for n in range(len(h)):
        assert _config(_write(tmp_path, h[:n]))[0] == -1, n


@pytest.mark.parametrize("field,value", [("sh_degree", 4), ("sh_degree", -1), ("width", 0), ("height", -5), ("world", 0),
                                         ("rank", 2), ("rank", -1), ("views_per_rank", 0), ("views_per_rank", 17), ("world", 9),
                                         ("capacity", 0), ("capacity", 1000), ("max_iters", 0)])
def test_out_of_range_config_is_refused(tmp_path, field, value):
    assert _config(_write(tmp_path, F.header(dict(CFG, **{field: value})) + F.END))[0] == -1


def test_missing_file_and_null_arguments_are_refused(tmp_path):
    from gaussian_lic_b200 import capi
    assert _config(tmp_path / "absent.ckpt")[0] == -1
    assert b"cannot open" in capi.lib.glic_last_error()
    cfg = capi.MapperConfig()
    assert capi.lib.glic_mapper_checkpoint_config(None, C.byref(cfg)) == -1
    assert capi.lib.glic_mapper_checkpoint_config(str(_write(tmp_path, F.header(CFG))).encode(), None) == -1


def test_python_mapper_reads_the_config(tmp_path):
    from gaussian_lic_b200 import mapper
    cfg = mapper.checkpoint_config(_write(tmp_path, F.header(CFG) + F.END))
    assert (cfg.width, cfg.height, cfg.capacity, cfg.seed, cfg.rank, cfg.world) == (320, 208, 4096, CFG["seed"], 1, 2)
