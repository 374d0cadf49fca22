#!/usr/bin/env python
"""What re-cutting connected strips costs and what it buys (nrdCudaRepartition): REBLUR_DIFFUSE_SPECULAR on 3840x2160 textures,
two strip contexts of this process (one GPU, arenas connected by pointer, as in tests/test_gpu_strips.py), stripHeight reserved
for a cut of a 1920x1080 rect.  Frames run at the full rect, then the rect drops to 1920x1080 and stays there.  The same run is done
twice: once keeping the first partition (rank 1's strip lies below the rect and launches nothing), once re-cutting the live rows
before the first small frame.  Reports, as one JSON line:

  repartition_ms_*      CUDA events on each rank's stream around nrdCudaRepartition: the first call (it also grows the
                        stream-ordered memory pool), then a second call with the same table
  bytes                 per rank, from texture shapes: "pulled", the rows the copy kernel reads (own and ghost rows of every
                        texture under the new table); "from_peer", the part another rank owned before; "copied_back", the
                        texture region of the arena (scratch -> arena)
  kernel_ms_small_rect  per rank: sum of nrdCudaGetTiming kernel times over the small-rect frames, kept vs re-cut

Both strips share the SMs of one GPU here, so this shows how the work is balanced between the ranks, not a speed-up.

    python tools/time_strips_repartition.py [--full-frames 3 --frames 10 --out profiles/strips_repartition.json]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

TILE = 16


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--width", type=int, default=3840)
    ap.add_argument("--height", type=int, default=2160)
    ap.add_argument("--small", type=int, nargs=2, default=[1920, 1080])
    ap.add_argument("--full-frames", type=int, default=3)
    ap.add_argument("--frames", type=int, default=10)
    ap.add_argument("--halo", type=int, default=96)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("time_strips_repartition.py needs a CUDA device")
    from time_reblur_passes import gpu_info
    from raytracingdenoiser_b200 import harness, nrd, scene, strips
    W, H = args.width, args.height
    sw, sh = args.small
    den = nrd.Denoiser.REBLUR_DIFFUSE_SPECULAR
    names = harness.denoiser_resources(den)
    halo = max(TILE, (args.halo + TILE - 1) // TILE * TILE)
    tiles = (H + TILE - 1) // TILE
    live = (sh + TILE - 1) // TILE
    _, first = strips.partition_rows_weighted(H, 2, [1.0] * tiles, min_rows=halo)
    # the capacity of the small-rect cut: half the live rows on rank 0, the rest of the frame on rank 1
    capacity = H - (live + 1) // 2 * TILE
    _, small_cut = strips.partition_rows_weighted(H, 2, [1.0 if t < live else 0.0 for t in range(tiles)], min_rows=halo, max_rows=capacity)
    out = {"denoiser": "REBLUR_DIFFUSE_SPECULAR", "size": [W, H], "small_rect": [sw, sh], "halo": halo, "strip_height": capacity,
           "first_partition": first, "small_rect_partition": small_cut, "full_frames": args.full_frames, "small_frames": args.frames,
           "note": "two strip contexts of one process share one GPU: kernel_ms shows the per-rank balance, not a speed-up; "
                   "frame time across GPUs is not measured"}
    out.update(gpu_info())
    scenes = {}
    for recut in (False, True):
        parts = [strips.StripDenoiser(den, W, H, r, 2, halo_rows=halo, partition=(capacity, first)) for r in range(2)]
        try:
            for p in parts:
                p.connect_local(parts)
            streams = [torch.cuda.Stream() for _ in parts]
            kernel_ms = [0.0, 0.0]
            for f in range(args.full_frames + args.frames):
                small = f >= args.full_frames
                rw, rh = (sw, sh) if small else (W, H)
                prev_h = sh if f > args.full_frames else H
                if (rw, rh) not in scenes:
                    scenes[(rw, rh)] = scene.Scene(rw, rh, device="cuda:0")
                fr = scenes[(rw, rh)].frame(f)
                if recut and f == args.full_frames:
                    # live rows: tiles(max(rectSize.y, rectSizePrev.y)) of the first small frame are still the full frame's; the cut
                    # is made for the small rect, which every later frame keeps
                    torch.cuda.synchronize()
                    events = []
                    for p, st in zip(parts, streams):
                        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        e0.record(st)
                        p.repartition(small_cut, st)
                        e1.record(st)
                        events.append((e0, e1))
                    torch.cuda.synchronize()
                    out["repartition_ms_first_call"] = [e0.elapsed_time(e1) for e0, e1 in events]
                    # the same table again: the same bytes move (every row from its own rank now), with the memory pool grown and
                    # both ranks' calls issued back to back
                    events = []
                    for p, st in zip(parts, streams):
                        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        e0.record(st)
                        p.repartition(small_cut, st)
                        e1.record(st)
                        events.append((e0, e1))
                    torch.cuda.synchronize()
                    out["repartition_ms_warm_call"] = [e0.elapsed_time(e1) for e0, e1 in events]
                    out["bytes"] = [_moved_bytes(p, parts[0].instance, W, H, halo, first, small_cut) for p in parts]
                canvas = {}
                for name in names:
                    if name.startswith("IN_"):
                        t = fr[name]
                        canvas[name] = torch.zeros((H, W) + tuple(t.shape[2:]), dtype=t.dtype, device=t.device)
                        canvas[name][:rh, :rw] = t
                cs = harness.make_common_settings(fr, rw, rh, f, common=dict(resourceSize=(W, H), resourceSizePrev=(W, H), rectSizePrev=(W if prev_h == H else sw, prev_h)))
                torch.cuda.synchronize()
                for p, st in zip(parts, streams):
                    p.set_input_strips({n: canvas[n][p.y0:p.y1] for n in canvas}, st)
                    p.ctx.set_timing(small)
                for p, st in zip(parts, streams):
                    p.denoise(cs, st)
                for r, (p, st) in enumerate(zip(parts, streams)):
                    p.synchronize(st)
                    if small:
                        kernel_ms[r] += sum(p.ctx.get_timing()[0])
            out["kernel_ms_small_rect_" + ("recut" if recut else "kept")] = kernel_ms
        finally:
            for p in parts:
                p.destroy()
    text = json.dumps(out)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        open(args.out, "w").write(text + "\n")


def _moved_bytes(part, instance, W, H, halo, old, new):
    """Per rank, from texture shapes: bytes the copy kernel reads (every row of the new window [y0 - halo, y1 + halo) inside the frame,
    of every arena texture), the part of them another rank owned before, and the texture region the copy back writes."""
    from raytracingdenoiser_b200 import nrd
    desc = instance.get_instance_desc()
    pitches = []  # (pitch, downsample) of every arena texture
    for kind, lst in ((nrd.ResourceType.PERMANENT_POOL, desc["permanentPool"]), (nrd.ResourceType.TRANSIENT_POOL, desc["transientPool"])):
        for i, (_, ds) in enumerate(lst):
            pitches.append((part.ctx.get_texture(kind, i).pitchBytes, ds))
    for name in nrd.ResourceType.__members__:
        if name.startswith(("IN_", "OUT_")):
            try:
                pitches.append((part.ctx.get_texture(getattr(nrd.ResourceType, name)).pitchBytes, 1))
            except nrd.NrdError:
                pass
    # the two kinds nrdCudaGetTexture does not expose: the decoded-guide surface (RGBA32F) and the staged copy of every guide input
    # (harness.RECT_ORIGIN_INPUTS, in the format of the input)
    from raytracingdenoiser_b200 import harness
    pad = lambda b: (W * b + 255) // 256 * 256  # noqa: E731
    pitches.append((pad(4 * 4), 1))
    for name in harness.RECT_ORIGIN_INPUTS:
        fmt = harness.user_format(nrd.Denoiser.REBLUR_DIFFUSE_SPECULAR, name)[0]
        pitches.append((pad(nrd.FORMAT_BYTES[nrd.Format(fmt)]), 1))
    y0, y1 = new[part.rank]
    o0, o1 = old[part.rank]
    pulled = from_peer = 0
    for pitch, ds in pitches:
        h = (H + ds - 1) // ds
        a, b = max(0, (y0 - halo) // ds), min(h, (y1 + halo + ds - 1) // ds)
        own_a, own_b = o0 // ds, (o1 + ds - 1) // ds
        pulled += (b - a) * pitch
        from_peer += ((b - a) - max(0, min(b, own_b) - max(a, own_a))) * pitch
    return {"pulled": pulled, "from_peer": from_peer, "copied_back": part.ctx.arena()[1] - 256}


if __name__ == "__main__":
    main()
