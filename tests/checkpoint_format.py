"""A restatement of the mapper checkpoint file of include/glic_b200.h ("Checkpoints") in numpy: the header writer the host tests
use, and a reader of a whole file the GPU tests check against the mapper's getters, so that the documented format and the one
the library writes cannot drift apart."""
import struct

import numpy as np

MAGIC = b"GLICCKPT"
VERSION = 1
HEADER_BYTES = 96
# the glic_mapper_config fields in the header's order, with their struct codes
CONFIG_FIELDS = [("width", "i"), ("height", "i"), ("fx", "f"), ("fy", "f"), ("cx", "f"), ("cy", "f"), ("sh_degree", "i"),
                 ("position_lr", "f"), ("feature_lr", "f"), ("opacity_lr", "f"), ("scaling_lr", "f"), ("rotation_lr", "f"),
                 ("lambda_dssim", "f"), ("scaling_scale", "f"), ("capacity", "I"), ("max_iters", "i"), ("seed", "Q"), ("rank", "i"),
                 ("world", "i"), ("views_per_rank", "i")]
CONFIG_FMT = "<" + "".join(c for _, c in CONFIG_FIELDS)
STATS_FIELDS = [("num_gaussians", "I"), ("capacity", "I"), ("iterations", "Q"), ("last_inserted", "I"), ("last_loss", "f"),
                ("mean_visible", "d"), ("overflow_regrows", "I"), ("ms_extend", "f"), ("ms_optimize", "f")]
SCHEDULE_FIELDS = [("densify_from", "I"), ("densify_until", "I"), ("densify_interval", "I"), ("opacity_reset_interval", "I"),
                   ("grad_threshold", "f"), ("percent_dense", "f"), ("min_opacity", "f"), ("reset_opacity", "f"), ("screen_radius", "i"),
                   ("world_scale_factor", "f"), ("scene_extent", "f")]
FLAGS = dict(initialized=1, exposure=2, pose=4, densification=8, frames=16)
GROUPS = [("rots", 4), ("means", 3), ("log_scales", 3), ("opacity_logits", 1), ("dc", 3), ("sh", None)]   # sh: 3 M floats per row
KEYFRAME_RECORD = 376


def header(cfg, magic=MAGIC, version=VERSION):
    """The 96-byte header of a configuration given as a dict of the glic_mapper_config fields"""
    return magic + struct.pack("<I", version) + struct.pack(CONFIG_FMT, *[cfg[k] for k, _ in CONFIG_FIELDS])


def section(tag, payload):
    return tag.encode() + struct.pack("<IQ", 0, len(payload)) + payload


END = section("END ", b"")


class _Cursor:
    def __init__(self, buf, off=0):
        self.buf, self.off = buf, off

    def take(self, fmt):
        v = struct.unpack_from("<" + fmt, self.buf, self.off)
        self.off += struct.calcsize("<" + fmt)
        return v if len(v) > 1 else v[0]

    def array(self, dtype, shape):
        n = int(np.prod(shape))
        a = np.frombuffer(self.buf, dtype, n, self.off).reshape(shape).copy()
        self.off += a.nbytes
        return a

    def fields(self, spec):
        return {k: self.take(c) for k, c in spec}


def sections(buf):
    """-> (config dict, [(tag, offset, length)] in file order); the end marker must end the file"""
    assert buf[:8] == MAGIC and struct.unpack_from("<I", buf, 8)[0] == VERSION
    cfg = dict(zip([k for k, _ in CONFIG_FIELDS], struct.unpack_from(CONFIG_FMT, buf, 12)))
    out, off = [], HEADER_BYTES
    while True:
        tag = buf[off:off + 4].decode()
        zero, n = struct.unpack_from("<IQ", buf, off + 4)
        assert zero == 0
        off += 16
        if tag == "END ":
            assert n == 0 and off == len(buf)
            return cfg, out
        out.append((tag, off, n))
        off += n


def read(path):
    """The whole file as a dict: config, and per section its fields and numpy arrays"""
    buf = open(path, "rb").read()
    cfg, secs = sections(buf)
    W, H, deg = cfg["width"], cfg["height"], cfg["sh_degree"]
    M = (deg + 1) ** 2 - 1
    out = dict(config=cfg, order=[t for t, _, _ in secs])
    for tag, off, n in secs:
        c = _Cursor(buf, off)
        if tag == "MAP ":
            P, Pcap, n_sky = c.take("III")
            arenas = []
            for _ in range(3):
                a = {}
                for name, w in GROUPS:
                    w = 3 * M if w is None else w
                    a[name] = c.array(np.float32, (P, w))
                arenas.append(a)
            out["map"] = dict(P=P, Pcap=Pcap, n_sky=n_sky, params=arenas[0], exp_avg=arenas[1], exp_avg_sq=arenas[2],
                              anchor=c.array(np.int32, (P,)))
        elif tag == "CNTR":
            d = dict(stats=c.fields(STATS_FIELDS))
            d["view_counter"], d["bin_cap"], d["binning_bytes"], d["sample_bytes"] = c.take("QqQQ")
            d["optimizer"], d["deterministic"], d["flags"], L = c.take("IIII")
            d["rng"] = bytes(buf[c.off:c.off + L]).decode()
            c.off += L
            out["counters"] = d
        elif tag == "KEYF":
            n_train, n_test = c.take("II")
            kfs = []
            for i in range(n_train + n_test):
                k = dict(train=i < n_train, R_wc=c.array(np.float32, (3, 3)), t_wc=c.array(np.float32, (3,)), cam=c.array(np.float32, (42,)),
                         cam_dev=c.array(np.float32, (36,)))
                k["kind"], k["frame"], k["mask_valid"], k["mask_valid_left"] = c.take("IIII")
                k["image"] = c.array(np.uint8, (H, W, 3)) if k["kind"] == 0 else c.array(np.float32, (3, H, W))
                if k["mask_valid"]:
                    words = c.array(np.uint32, (H, (W + 31) // 32))
                    bits = (words[:, np.arange(W) >> 5] >> (np.arange(W) & 31).astype(np.uint32)) & 1
                    k["mask"] = bits.astype(np.uint8)
                kfs.append(k)
            out["keyframes"] = dict(n_train=n_train, n_test=n_test, list=kfs)
        elif tag == "EXPO":
            lr, k = c.take("fI")
            out["exposure"] = dict(lr=lr, n=k, E=c.array(np.float32, (k, 3, 4)), m=c.array(np.float32, (k, 3, 4)),
                                   v=c.array(np.float32, (k, 3, 4)), t=c.array(np.int32, (k,)))
        elif tag == "POSE":
            lr_rho, lr_omega, k = c.take("ffI")
            out["pose"] = dict(lr_rho=lr_rho, lr_omega=lr_omega, n=k, T=c.array(np.float64, (k, 12)), f=c.array(np.float32, (k, 12)),
                               m=c.array(np.float32, (k, 6)), v=c.array(np.float32, (k, 6)), t=c.array(np.int32, (k,)))
        elif tag == "DENS":
            calls, P = c.take("QI")
            out["densification"] = dict(calls=calls, accum=c.array(np.float32, (P,)), denom=c.array(np.float32, (P,)),
                                        maxr=c.array(np.int32, (P,)))
        elif tag == "SCHD":
            on = c.take("I")
            s = c.fields(SCHEDULE_FIELDS)
            t = c.fields([("cloned", "I"), ("split", "I"), ("pruned", "I"), ("rows", "I")])
            steps, resets = c.take("II")
            out["schedule"] = dict(on=on, schedule=s, totals=t, steps=steps, resets=resets)
        elif tag == "FRMS":
            k, sky_points, sky_radius = c.take("iii")
            st = c.fields([("frames", "I"), ("train", "I"), ("test", "I"), ("pending_points", "I"), ("image_bytes", "Q")])
            p = st["pending_points"]
            out["frames"] = dict(k=k, sky_points=sky_points, sky_radius=sky_radius, stats=st, xyz=c.array(np.float32, (p, 3)),
                                 rgb=c.array(np.uint8, (p, 3)), depth=c.array(np.float32, (p,)))
        else:
            raise AssertionError("unknown section %r" % tag)
        assert c.off == off + n, "section %s: %d bytes parsed of %d" % (tag, c.off - off, n)
    return out


def packed_moments(arena, M):
    """an arena's groups in download(moments=True)'s packed order (rot, xyz, log-scale, opacity, dc, sh-rest), flat"""
    return np.concatenate([np.ravel(arena[name]) for name, _ in GROUPS])
