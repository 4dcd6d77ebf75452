"""LPIPS (AlexNet) weights: the TorchScript lpips_alex.pt of Gaussian-LIC -> the flat file glic_lpips reads.

Plumbing only (torch is allowed here; the library itself reads the flat file without torch).  File layout (little-endian):
uint32 magic "LPIP", uint32 version 1, uint32 float count, uint32 0, then the floats
    mean[3] std[3] | conv0 OIHW weight, bias | conv3 .. | conv6 .. | conv8 .. | conv10 .. | lin0 .. lin4 (C floats each)
"""
import ctypes as C
import struct

import numpy as np

MAGIC = 0x5049504C          # b"LPIP"
VERSION = 1
CONVS = (0, 3, 6, 8, 10)    # indices of the conv layers in the traced net.layers


def state_keys():
    """state-dict keys in file order"""
    keys = ["net.mean", "net.std"]
    for i in CONVS:
        keys += ["net.layers.%d.weight" % i, "net.layers.%d.bias" % i]
    return keys + ["lin.%d.1.weight" % k for k in range(5)]


def payload(state):
    """flat float32 payload of a state dict (tensors or arrays)"""
    parts = []
    for k in state_keys():
        v = state[k]
        v = v.detach().cpu().numpy() if hasattr(v, "detach") else np.asarray(v)
        parts.append(np.ascontiguousarray(v, dtype=np.float32).reshape(-1))
    return np.concatenate(parts)


def load_state(pt_path):
    """state dict of the TorchScript module, on the CPU (its traced forward hard-codes cuda:0, the parameters do not)"""
    import torch
    return {k: v for k, v in torch.jit.load(str(pt_path), map_location="cpu").state_dict().items()}


def write(path, floats):
    f = np.ascontiguousarray(floats, dtype="<f4")
    with open(path, "wb") as out:
        out.write(struct.pack("<4I", MAGIC, VERSION, f.size, 0))
        out.write(f.tobytes())


def convert(pt_path, out_path):
    """lpips_alex.pt -> flat weight file; returns the payload"""
    p = payload(load_state(pt_path))
    write(out_path, p)
    return p


def read(path):
    """the payload through the library's own reader (glic_lpips_read_weights)"""
    from . import capi
    out = np.empty(int(capi.lib.glic_lpips_weight_floats()), np.float32)
    capi.check(capi.lib.glic_lpips_read_weights(str(path).encode(), out.ctypes.data_as(C.c_void_p)), "lpips_read_weights")
    return out


if __name__ == "__main__":
    import sys
    n = convert(sys.argv[1], sys.argv[2]).size
    print("%s: %d floats" % (sys.argv[2], n))
