"""Times every supported denoiser chain on one GPU (CUDA events, device-resident inputs, steady state) and prints one JSON
line per chain with the per-pass breakdown.  bench.py measures the headline metric; this is the evidence for the others.

    python tools/time_chains.py [--width 3840 --height 2160 --frames 16 --warmup 8] [--only NAME,...] [--digest]

--digest adds byte digests (tools/time_reblur_passes.py) of every output texture after every frame and, on the frames timed pass
by pass, of every texture each pass writes: compare the lines of two library builds (NRD_B200_LIB) to show that they compute the
same bytes.  The copies change what the passes find in L2, so take times from runs without it.
"""
import argparse
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--width", type=int, default=3840)
    ap.add_argument("--height", type=int, default=2160)
    ap.add_argument("--frames", type=int, default=16)
    ap.add_argument("--warmup", type=int, default=8)
    ap.add_argument("--only", default="")
    ap.add_argument("--digest", action="store_true")
    args = ap.parse_args()
    import torch
    from raytracingdenoiser_b200 import build
    build.build_all()
    from raytracingdenoiser_b200 import harness, nrd, scene
    from time_reblur_passes import Digests
    W, H = args.width, args.height
    dev = torch.device("cuda", 0)
    stream = torch.cuda.current_stream(dev)
    for den in (nrd.Denoiser.REBLUR_DIFFUSE, nrd.Denoiser.REBLUR_SPECULAR, nrd.Denoiser.REBLUR_DIFFUSE_SPECULAR, nrd.Denoiser.RELAX_DIFFUSE_SPECULAR,
                nrd.Denoiser.SIGMA_SHADOW, nrd.Denoiser.SIGMA_SHADOW_TRANSLUCENCY):
        if args.only and den.name not in args.only.split(","):
            continue
        sc = scene.Scene(W, H, device="cuda:0")
        mode = harness.radiance_mode(den)
        frames = [sc.frame(f, mode) for f in range(args.warmup + args.frames)]
        gpu = harness.GpuDenoiser(den, W, H)
        dg = Digests(gpu.ctx, stream)
        frame_digests = []

        def record(digests):
            if args.digest:
                digests.update({name: dg.tensor(t) for name, t in gpu.outputs().items()})
                frame_digests.append(Digests.hex(digests))

        for i in range(args.warmup):
            gpu.set_inputs(frames[i])
            gpu.denoise(harness.make_common_settings(frames[i], W, H, i))
            record({})
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        total, per_pass = 0.0, {}
        pipelines = gpu.instance.get_instance_desc()["pipelines"]
        for i in range(args.warmup, args.warmup + args.frames):
            gpu.set_inputs(frames[i])
            cs = harness.make_common_settings(frames[i], W, H, i)
            if i % 2 == 0:   # whole-chain time
                e0.record(stream)
                gpu.denoise(cs)
                e1.record(stream)
                torch.cuda.synchronize()
                total += e0.elapsed_time(e1)
                record({})
            else:            # per-pass breakdown
                gpu.instance.set_common_settings(cs)
                r, raw, n = gpu.instance.get_compute_dispatches_raw([gpu.identifier])
                evs, digests = [], {}
                for j in range(n):
                    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    a.record(stream)
                    gpu.ctx.execute_raw(C.byref(raw[j]), stream.cuda_stream)
                    b.record(stream)
                    evs.append((raw[j].name.decode().split(" - ")[-1], a, b))
                    if args.digest:
                        for dt, rt, idx in nrd.Dispatch(raw[j], pipelines).resources:
                            if dt == nrd.DescriptorType.STORAGE_TEXTURE:
                                digests["%d %s:%s[%d]" % (j, evs[-1][0], rt.name, idx)] = dg.texture(rt, idx)
                torch.cuda.synchronize()
                for name, a, b in evs:
                    per_pass.setdefault(name, []).append(a.elapsed_time(b))
                record(digests)
        nwhole = (args.frames + 1) // 2
        ms = total / nwhole
        print(json.dumps({"denoiser": den.name, "size": [W, H], "ms_per_frame": round(ms, 3), "mpixels_per_s": round(W * H / ms / 1e3, 1),
                          "per_pass_ms": {k: round(sum(v) / len(v) * (v and 1), 3) for k, v in per_pass.items()},
                          "passes_per_frame": {k: round(len(v) / (args.frames // 2), 1) for k, v in per_pass.items()},
                          **({"digests": frame_digests} if args.digest else {})}))
        gpu.destroy()
        del frames, gpu
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
