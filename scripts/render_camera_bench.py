"""Cost of rendering from any camera at cfg2 (500 k Gaussians, 1920x1080, SH degree 3).

  - the blend kernel alone (render_forward_kernel, GLIC_STAGE_RENDER_FWD events of glic_profile): the training form under
    glic_forward against the inference form under glic_render, windows alternating in this one process;
  - a whole frame: glic_forward against glic_render (CUDA events around `--frames` back-to-back calls per window, profiling
    off), with the size of the checkpoint buffer the training form needs and the inference form does not;
  - glic_mapper_render_camera on a native mapper of the same map: host clock around the synchronising call at 1920x1080 and
    3840x2160, with the four outputs in host memory and in device memory.

    python scripts/render_camera_bench.py [--config cfg2] [--windows 7] [--frames 20]

Prints one JSON line with the medians, every window, and the card name and power limit.  Needs a GPU; writes nothing."""
import argparse
import ctypes as C
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="cfg2")
    ap.add_argument("--windows", type=int, default=7)
    ap.add_argument("--frames", type=int, default=20, help="calls per timed window")
    args = ap.parse_args()
    import numpy as np
    import torch
    from gaussian_lic_b200 import capi, mapper as gmapper, model, ops, synthetic as syn
    from pose_bench import card
    assert torch.cuda.is_available(), "render_camera_bench.py needs a GPU"
    P, W, H, fx, fy, cx, cy, deg, _ = syn.CONFIGS[args.config]
    g, _ = syn.make_scene(args.config)
    dev = torch.device("cuda:0")
    mdl = model.PackedModel(dict(g, degree=deg), dev)
    mdl.activate()
    gi = mdl.inputs
    R_wc, t_wc = syn.orbit_pose(1, radius=0.25)
    cam = gmapper.camera_block(W, H, fx, fy, cx, cy, R_wc, t_wc)
    rast = ops.CRasterizer(W, H, dev)
    view = rast.make_view(cam)
    color, T, radii = rast.forward(gi, view)                  # sizes the workspaces (both calls share them)
    ren = rast.render(gi, view, radii=radii)
    same = bool(torch.equal(color.view(torch.int32), ren["color"].view(torch.int32)) and
                torch.equal(T.view(torch.int32), ren["final_T"].view(torch.int32)))
    R_pairs, B = rast.R, rast.B
    lib, M = capi.lib, rast.M
    f32 = dict(dtype=torch.float32, device=dev)
    depth, median = torch.empty(H, W, **f32), torch.empty(H, W, **f32)

    def common():
        return (P, deg, M, capi.ptr(gi["means"]), capi.ptr(gi["scales"]), 1.0, capi.ptr(gi["rots"]), capi.ptr(gi["opacity"]),
                capi.ptr(gi["dc"]), capi.ptr(gi["sh"]) if M else None, C.byref(view))

    def forward():
        capi.check(lib.glic_forward(*common(), 0, capi.ptr(radii), capi.ptr(rast.geom_ws), rast.geom_ws.numel(), capi.ptr(rast.image_ws),
                                    rast.image_ws.numel(), capi.ptr(rast.binning_ws), rast.binning_ws.numel(), capi.ptr(rast.sample_ws),
                                    rast.sample_ws.numel(), capi.ptr(color), capi.ptr(T), None, None), "forward")

    def render():
        capi.check(lib.glic_render(*common(), capi.ptr(radii), capi.ptr(rast.geom_ws), rast.geom_ws.numel(), capi.ptr(rast.image_ws),
                                   rast.image_ws.numel(), capi.ptr(rast.binning_ws), rast.binning_ws.numel(), capi.ptr(color), capi.ptr(T),
                                   capi.ptr(depth), capi.ptr(median), None, None), "render")

    calls = {"training": forward, "inference": render}
    for fn in calls.values():
        for _ in range(5):
            fn()
    torch.cuda.synchronize()
    # the blend kernel alone, by the library's stage events
    blend = {k: [] for k in calls}
    for _ in range(args.windows):
        for k, fn in calls.items():
            torch.cuda.synchronize()
            capi.profile_enable(True)
            for _ in range(args.frames):
                fn()
            torch.cuda.synchronize()
            ms, n = capi.profile_read()["render_fwd"]
            capi.profile_enable(False)
            blend[k].append(1e3 * ms / n)
    # whole frames, profiling off
    frame = {k: [] for k in calls}
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    for _ in range(args.windows):
        for k, fn in calls.items():
            torch.cuda.synchronize()
            ev[0].record()
            for _ in range(args.frames):
                fn()
            ev[1].record()
            torch.cuda.synchronize()
            frame[k].append(ev[0].elapsed_time(ev[1]) / args.frames)

    # the mapper call, host clock (it ends in a synchronise)
    m = gmapper.Mapper(W, H, fx, fy, cx, cy, sh_degree=deg, capacity=P)
    m.initialize(g)
    host = {}
    for Wf, Hf in ((1920, 1080), (3840, 2160)):                  # the configured field of view at both sizes
        name = "%dx%d" % (Wf, Hf)
        k = dict(width=Wf, height=Hf, fx=fx * Wf / W, fy=fy * Hf / H, cx=Wf / 2.0, cy=Hf / 2.0)
        rc = capi.RenderCamera()
        rc.R_wc[:] = [float(x) for x in np.asarray(R_wc, np.float32).reshape(9)]
        rc.t_wc[:] = [float(x) for x in np.asarray(t_wc, np.float32).reshape(3)]
        rc.fx, rc.fy, rc.cx, rc.cy, rc.width, rc.height = k["fx"], k["fy"], k["cx"], k["cy"], Wf, Hf
        outs = {"host": [np.empty(n, np.float32) for n in (3 * Wf * Hf, Wf * Hf, Wf * Hf, Wf * Hf)],
                "device": [torch.empty(n, **f32) for n in (3 * Wf * Hf, Wf * Hf, Wf * Hf, Wf * Hf)]}
        ptrs = {"host": [a.ctypes.data_as(C.c_void_p) for a in outs["host"]], "device": [capi.ptr(t) for t in outs["device"]]}
        for where in ptrs:
            capi.check(lib.glic_mapper_render_camera(m._h, C.byref(rc), -1, 1, *ptrs[where]), "mapper_render_camera")
        for where in ptrs:
            ts = []
            for _ in range(args.windows):
                t0 = time.perf_counter()
                capi.check(lib.glic_mapper_render_camera(m._h, C.byref(rc), -1, 1, *ptrs[where]), "mapper_render_camera")
                ts.append(1e3 * (time.perf_counter() - t0))
            host["%s_%s" % (name, where)] = ts
    m.close()
    med = lambda v: float(np.median(v))       # noqa: E731
    ckpt_bytes = B * 256 * 16                 # the training form's checkpoint buffer for this frame (it writes the part its pixels reach)
    out = {"config": args.config, "P": P, "W": W, "H": H, "R": R_pairs, "buckets": B, "windows": args.windows, "frames": args.frames,
           "colour_and_T_bit_identical": same,
           "blend_us": {k: round(med(v), 2) for k, v in blend.items()},
           "frame_ms": {k: round(med(v), 4) for k, v in frame.items()},
           "checkpoint_buffer_bytes": ckpt_bytes,
           "mapper_render_camera_ms": {k: round(med(v), 3) for k, v in host.items()},
           "window_blend_us": {k: [round(x, 2) for x in v] for k, v in blend.items()},
           "window_frame_ms": {k: [round(x, 4) for x in v] for k, v in frame.items()},
           "window_mapper_ms": {k: [round(x, 3) for x in v] for k, v in host.items()},
           "card": card()}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
