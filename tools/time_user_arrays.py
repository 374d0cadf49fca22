"""Cost of binding user textures as CUDA arrays (nrdCudaSetUserTextureArray) instead of device pointers: 4K
REBLUR_DIFFUSE_SPECULAR in steady state, one context with every user texture bound by pointer and one with every user texture bound
as a CUDA array, on the same frames, alternating frame by frame.  Prints one JSON line:

  frame_ms_pointer / frame_ms_array   CUDA events around nrdCudaDenoise (median and mean over the timed frames)
  conversion_ms                       ArrayToShadowKernel + ShadowToArrayKernel per frame, from torch.profiler in a run of its own
  conversion_bytes                    what the two launches must move, from the formats: array + shadow bytes of every input
                                      converted in and of every texture the frame's passes write, converted back
  gpu, power_limit_w                  read in the same run

    python tools/time_user_arrays.py [--width 3840 --height 2160 --frames 24 --warmup 8] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"], capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("nvidia-smi: %s" % r.stderr)
    name, limit = [s.strip() for s in r.stdout.strip().splitlines()[0].split(",")]
    return name, float(limit)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--width", type=int, default=3840)
    ap.add_argument("--height", type=int, default=2160)
    ap.add_argument("--frames", type=int, default=24)
    ap.add_argument("--warmup", type=int, default=8)
    ap.add_argument("--profiled", type=int, default=4)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    import torch
    from raytracingdenoiser_b200 import build
    build.build_all()
    from raytracingdenoiser_b200 import harness, nrd, scene
    from raytracingdenoiser_b200.cuda_arrays import CudaArray
    assert torch.cuda.is_available(), "this measurement needs a CUDA device"
    W, H = args.width, args.height
    den = nrd.Denoiser.REBLUR_DIFFUSE_SPECULAR
    dev = torch.device("cuda", 0)
    stream = torch.cuda.current_stream(dev).cuda_stream
    sc = scene.Scene(W, H, device="cuda:0")
    n_frames = args.warmup + args.frames + args.profiled
    frames = [sc.frame(f, harness.radiance_mode(den)) for f in range(n_frames)]

    pointer = harness.GpuDenoiser(den, W, H)
    inst = nrd.Instance([(0, den)])
    ctx = nrd.CudaContext(inst, W, H)
    names = harness.denoiser_resources(den)
    arrays = {}
    for name in names:
        fmt = harness.user_format(den, name)[0]
        arrays[name] = CudaArray(fmt, W, H)
        ctx.set_user_texture_array(getattr(nrd.ResourceType, name), arrays[name].handle.value, fmt)

    def array_frame(f, fr, timed=None):
        for name in names:
            if name.startswith("IN_"):
                arrays[name].upload(fr[name])
        inst.set_common_settings(harness.make_common_settings(fr, W, H, f))
        if timed:
            timed[0].record()
        ctx.denoise([0], stream=stream)
        if timed:
            timed[1].record()

    def pointer_frame(f, fr, timed=None):
        pointer.set_inputs(fr)
        pointer.instance.set_common_settings(harness.make_common_settings(fr, W, H, f))
        if timed:
            timed[0].record()
        pointer.ctx.denoise([0], stream=stream)
        if timed:
            timed[1].record()

    for f in range(args.warmup):
        pointer_frame(f, frames[f])
        array_frame(f, frames[f])
    torch.cuda.synchronize()
    times = {"pointer": [], "array": []}
    for f in range(args.warmup, args.warmup + args.frames):
        for kind, run in (("pointer", pointer_frame), ("array", array_frame)):
            ev = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
            run(f, frames[f], ev)
            torch.cuda.synchronize()
            times[kind].append(ev[0].elapsed_time(ev[1]))
    # the two outputs must agree: the array path is a copy around the same kernels
    for name in names:
        if name.startswith("OUT_") or name == "IN_MV":
            _, dtype, ch = harness.user_format(den, name)
            assert torch.equal(arrays[name].download(dtype, ch), pointer.tex[name]), "%s differs between the bindings" % name

    # conversion launches alone, in a profiled run of their own
    from torch.profiler import ProfilerActivity, profile
    first = args.warmup + args.frames
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for f in range(first, first + args.profiled):
            array_frame(f, frames[f])
        torch.cuda.synchronize()
    conv = {"ArrayToShadowKernel": 0.0, "ShadowToArrayKernel": 0.0}
    launches = 0
    for e in prof.events():
        for k in conv:
            if k in e.name and e.device_type.name == "CUDA":
                conv[k] += e.device_time_total / 1000.0
                launches += 1
    if not launches:
        raise RuntimeError("the profiler saw no conversion kernel")

    # algorithmic bytes: every input in (array read + shadow write), every texture a pass of a steady-state frame writes back
    inst.set_common_settings(harness.make_common_settings(frames[first], W, H, first))
    written = {rt.name for d in inst.get_compute_dispatches([0]) for dt, rt, _ in d.resources if dt == nrd.DescriptorType.STORAGE_TEXTURE}
    per_px = lambda subset: sum(2 * nrd.FORMAT_BYTES[harness.user_format(den, n)[0]] for n in subset)
    in_px = per_px([n for n in names if n.startswith("IN_")])
    back_px = per_px([n for n in names if n in written])
    conv_bytes = (in_px + back_px) * W * H
    conv_ms = (conv["ArrayToShadowKernel"] + conv["ShadowToArrayKernel"]) / args.profiled
    name, limit = card()
    med = lambda v: sorted(v)[len(v) // 2]
    result = {
        "metric": "user_arrays_%s_%dx%d" % (den.name, W, H), "gpu": name, "power_limit_w": limit, "frames": args.frames,
        "frame_ms_pointer": {"median": round(med(times["pointer"]), 4), "mean": round(sum(times["pointer"]) / len(times["pointer"]), 4)},
        "frame_ms_array": {"median": round(med(times["array"]), 4), "mean": round(sum(times["array"]) / len(times["array"]), 4)},
        "conversion_ms": {"in": round(conv["ArrayToShadowKernel"] / args.profiled, 4), "back": round(conv["ShadowToArrayKernel"] / args.profiled, 4),
                          "total": round(conv_ms, 4), "launches_per_frame": launches / args.profiled},
        "conversion_bytes": {"in_per_px": in_px, "back_per_px": back_px, "per_frame": conv_bytes, "written_back": sorted(n for n in names if n in written)},
        "conversion_gb_per_s": round(conv_bytes / (conv_ms * 1e-3) / 1e9, 1),
    }
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(line + "\n")
    pointer.destroy()
    ctx.destroy()
    inst.destroy()
    for a in arrays.values():
        a.destroy()


if __name__ == "__main__":
    main()
