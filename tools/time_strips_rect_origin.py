#!/usr/bin/env python
"""What staging the guide inputs costs connected strips under rectOrigin.y != 0 (executor.cu StagesInputs): REBLUR_DIFFUSE_SPECULAR
with isBaseColorMetalnessAvailable on two strip contexts of this process (one GPU, arenas connected by pointer, as in
tests/test_gpu_strips.py), a rect inside 3840x2160 textures at a non-zero origin.  Every frame runs the application-driven path
(SetCommonSettings, nrdCudaBarrier, the dispatch list) with nrdCudaSetTiming on, and reports per rank and frame:

  gather_ms          GatherRectOriginKernel (frame start: the guide inputs into their staged copies)
  gather_barrier_ms  the barrier after it
  pull_ms            PullRectOriginKernel (IN_MV back from the staged copy after REBLUR temporal stabilization)
  slots_ms           the sum of every timed slot of the frame: kernels, ghost pushes and barrier waits (clears are not timed)
  frame_ms           CUDA events on the rank's stream around the whole frame, frame-start barrier included

Both strips share one GPU here, so their kernels compete for the SMs and peer loads are HBM loads, not NVLink.

    python tools/time_strips_rect_origin.py [--frames 20 --warmup 5 --rect 3200 1800 --origin 320 180]
"""
import argparse
import ctypes as C
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--width", type=int, default=3840)
    ap.add_argument("--height", type=int, default=2160)
    ap.add_argument("--rect", type=int, nargs=2, default=[3200, 1800])
    ap.add_argument("--origin", type=int, nargs=2, default=[320, 180])
    ap.add_argument("--frames", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--halo", type=int, default=96)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("time_strips_rect_origin.py needs a CUDA device")
    from time_reblur_passes import gpu_info
    from raytracingdenoiser_b200 import harness, nrd, scene, strips
    W, H = args.width, args.height
    (rw, rh), (ox, oy) = args.rect, args.origin
    if args.origin[1] == 0 or ox + rw > W or oy + rh > H:
        raise SystemExit("the rect must fit the textures and have rectOrigin.y != 0 (the frames that stage)")
    den = nrd.Denoiser.REBLUR_DIFFUSE_SPECULAR
    flags = {"isBaseColorMetalnessAvailable": True}
    names = harness.denoiser_resources(den, flags)
    parts = [strips.StripDenoiser(den, W, H, r, 2, halo_rows=args.halo) for r in range(2)]
    for p in parts:
        p.connect_local(parts)
    streams = [torch.cuda.Stream() for _ in parts]
    sc = scene.Scene(rw, rh, device="cuda:0")
    pipelines = parts[0].instance.get_instance_desc()["pipelines"]
    canvas = {}  # the application's resource-sized G-buffer: guide inputs at rectOrigin, the noisy signals at (0, 0)
    rows = {r: [] for r in range(len(parts))}
    for p in parts:
        p.ctx.set_timing(True)
    for f in range(args.warmup + args.frames):
        fr = sc.frame(f)
        for name in names:
            if name.startswith("IN_"):
                t = fr[name]
                if name not in canvas:
                    canvas[name] = torch.zeros((H, W) + tuple(t.shape[2:]), dtype=t.dtype, device=t.device)
                x, y = (ox, oy) if name in harness.RECT_ORIGIN_INPUTS else (0, 0)
                canvas[name][y:y + rh, x:x + rw] = t
        cs = harness.make_common_settings(fr, rw, rh, f, common=dict(flags, resourceSize=(W, H), resourceSizePrev=(W, H), rectOrigin=(ox, oy)))
        torch.cuda.synchronize()
        events, lists = [], []
        for p, st in zip(parts, streams):
            p.set_input_strips({n: canvas[n][p.y0:p.y1] for n in names if n.startswith("IN_")}, st)
            lists.append(p.dispatches(cs))
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(st)
            p.ctx.barrier(st.cuda_stream)
            events.append((e0, e1))
        raw0, n = lists[0]
        for i in range(n):
            for p, st, (raw, _) in zip(parts, streams, lists):
                p.ctx.execute_raw(C.byref(raw[i]), st.cuda_stream)
        for (e0, e1), st in zip(events, streams):
            e1.record(st)
        for p, st in zip(parts, streams):
            p.synchronize(st)
        # timed slots: the gather, then every dispatch but the clears, the pull right after temporal stabilization
        labels = ["gather"]
        for i in range(n):
            d = nrd.Dispatch(raw0[i], pipelines)
            if d.shaderFileName.startswith("Clear_"):
                continue
            labels.append(d.name)
            if "TemporalStabilization" in d.shaderFileName:
                labels.append("pull")
        for r, (p, (e0, e1)) in enumerate(zip(parts, events)):
            kernel_ms, exchange_ms = p.ctx.get_timing()
            if len(kernel_ms) != len(labels):
                raise RuntimeError("rank %d: %d timed slots for %d labels" % (r, len(kernel_ms), len(labels)))
            if f >= args.warmup:
                rows[r].append({"gather_ms": kernel_ms[labels.index("gather")], "gather_barrier_ms": exchange_ms[labels.index("gather")],
                                "pull_ms": kernel_ms[labels.index("pull")], "slots_ms": sum(kernel_ms) + sum(exchange_ms), "frame_ms": e0.elapsed_time(e1)})
    for p in parts:
        p.ctx.set_timing(False)
        p.destroy()
    out = {"denoiser": "REBLUR_DIFFUSE_SPECULAR", "size": [W, H], "rect": [rw, rh], "origin": [ox, oy], "strips": [[p.y0, p.y1] for p in parts],
           "halo": args.halo, "frames": args.frames, "warmup": args.warmup, "isBaseColorMetalnessAvailable": True}
    out.update(gpu_info())
    for r, frames in rows.items():
        med = {k: statistics.median(x[k] for x in frames) for k in frames[0]}
        med["staging_share_of_frame"] = (med["gather_ms"] + med["gather_barrier_ms"] + med["pull_ms"]) / med["frame_ms"]
        out["rank%d_median" % r] = med
    text = json.dumps(out, indent=1)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        open(args.out, "w").write(text)


if __name__ == "__main__":
    main()
