"""Dynamic resolution in strip mode (the multi-GPU data path on ONE GPU, as in test_gpu_strips.py): the passes run over a rect
smaller than the textures, its size changes between frames (rectSizePrev != rectSize) and it sits at a rectOrigin of the guide
inputs.  After every frame every output -- and IN_MV, which REBLUR temporal stabilization patches when
isBaseColorMetalnessAvailable is set -- must be bit-identical to one full-frame context running the strip build of the kernels.
The scene is rendered at the rect size and placed into resource-sized inputs like an application's G-buffer: the guide inputs
at rectOrigin, the noisy signals at (0, 0) (Common.hlsli:200-205 WithRectOrigin)."""
import ctypes as C

import pytest

pytestmark = pytest.mark.gpu

W, H = 320, 192

# rect schedules: frame -> (originX, originY, width, height)
SCHEDULES = {
    "constant": lambda f: (0, 0, 250, 141),
    "shrink_grow": lambda f: [(0, 0, 320, 192), (0, 0, 250, 141), (0, 0, 160, 90), (0, 0, 280, 158), (0, 0, 320, 192)][f],
    # rows 0..39 (whole tiles: 48) lie in the first strip of every partition below: the other ranks launch nothing, after a
    # full frame that left data in their rows
    "first_strip_only": lambda f: [(0, 0, 320, 192), (0, 0, 200, 40), (0, 0, 200, 40), (0, 0, 230, 44), (0, 0, 200, 40)][f],
    # oy = 37: beyond a halo of 16 or 32 rows and not a whole tile; from frame 0, so the frame-0 clear of IN_MV is staged too
    "origin": lambda f: (24, 37, 250, 141),
    "moving_origin": lambda f: [(0, 0, 250, 141), (24, 37, 250, 141), (16, 8, 280, 158), (8, 50, 200, 120), (0, 0, 250, 141)][f],
}


def _placed_frame(scenes, mode, f, schedule):
    """(frame of resource-sized tensors, CommonSettings) of frame f; scenes caches one scene per rect size."""
    import torch
    from raytracingdenoiser_b200 import harness, scene
    ox, oy, rw, rh = schedule(f)
    prev = schedule(f - 1) if f > 0 else (ox, oy, rw, rh)
    if (rw, rh) not in scenes:
        scenes[(rw, rh)] = scene.Scene(rw, rh)
    fr = scenes[(rw, rh)].frame(f, mode)
    placed = dict(fr)
    for name, t in fr.items():
        if not (name.startswith("IN_") and torch.is_tensor(t)):
            continue
        full = torch.zeros((H, W) + tuple(t.shape[2:]), dtype=t.dtype, device=t.device)
        x, y = (ox, oy) if name in harness.RECT_ORIGIN_INPUTS else (0, 0)
        full[y:y + rh, x:x + rw] = t
        placed[name] = full
    common = dict(resourceSize=(W, H), resourceSizePrev=(W, H), rectSizePrev=(prev[2], prev[3]), rectOrigin=(ox, oy))
    return placed, common


def _copy_rows(part, name, tensor, to_context, stream):
    from raytracingdenoiser_b200 import nrd
    t = tensor[part.y0:part.y1]
    part.ctx.copy(getattr(nrd.ResourceType, name), 0, t.data_ptr(), t.stride(0) * t.element_size(), to_context, stream.cuda_stream)


def _run(denoiser_name, world, halo, schedule, whole_frame_call, base_color=False, weighted=False, frames=5):
    import os
    os.environ["NRD_B200_FORCE_STRIP_KERNELS"] = "1"  # the full-frame reference runs the strip build of the kernels
    try:
        _run_inner(denoiser_name, world, halo, SCHEDULES[schedule], whole_frame_call, base_color, weighted, frames)
    finally:
        del os.environ["NRD_B200_FORCE_STRIP_KERNELS"]


def _run_inner(denoiser_name, world, halo, schedule, whole_frame_call, base_color, weighted, frames):
    import torch
    from raytracingdenoiser_b200 import harness, nrd, scene, strips
    den = getattr(nrd.Denoiser, denoiser_name)
    mode = harness.radiance_mode(den)
    flags = {"isBaseColorMetalnessAvailable": True} if base_color else {}
    settings = None
    if base_color:  # thresholds low enough that the motion-vector patch rewrites part of IN_MV (as in test_gpu_reblur.py)
        settings = nrd.ReblurSettings()
        settings.specularProbabilityThresholdsForMvModification[0], settings.specularProbabilityThresholdsForMvModification[1] = 0.2, 0.6
    full = harness.GpuDenoiser(den, W, H, settings=settings, common=flags)
    partition = None
    if weighted:  # cost-balanced, non-uniform strips
        cost = strips.tile_row_cost_from_viewz(scene.Scene(W, H).frame(0, mode)["IN_VIEWZ"])
        partition = strips.partition_rows_weighted(H, world, cost, min_rows=max(halo, 16))
        assert len(set(y1 - y0 for y0, y1 in partition[1])) > 1, partition
    parts = [strips.StripDenoiser(den, W, H, r, world, halo_rows=halo, partition=partition, settings=settings) for r in range(world)]
    names = harness.denoiser_resources(den, flags)
    try:  # a failing case must not leak its strip-mode contexts (there are only kMaxPeerSlots per process)
        for p in parts:
            p.connect_local(parts)
        streams = [torch.cuda.Stream() for _ in parts]
        scenes = {}
        patched = False
        for f in range(frames):
            fr, common = _placed_frame(scenes, mode, f, schedule)
            common.update(flags)
            ox, oy, rw, rh = schedule(f)
            cs = harness.make_common_settings(fr, rw, rh, f, common=common)
            full.set_inputs(fr)
            full.denoise(cs)
            torch.cuda.synchronize()
            for p, st in zip(parts, streams):
                for name in names:
                    if name.startswith("IN_"):
                        _copy_rows(p, name, fr[name], True, st)
            if whole_frame_call:
                for p, st in zip(parts, streams):
                    p.denoise(cs, st)
            else:
                # the application-driven path: SetCommonSettings, then nrdCudaBarrier (it stages the guide inputs for this
                # rectOrigin), then the dispatch list, ranks interleaved pass by pass
                lists = []
                for p, st in zip(parts, streams):
                    lists.append(p.dispatches(cs))
                    p.ctx.barrier(st.cuda_stream)
                n = lists[0][1]
                assert all(m == n for _, m in lists)
                for i in range(n):
                    for p, st, (raw, _) in zip(parts, streams, lists):
                        p.ctx.execute_raw(C.byref(raw[i]), st.cuda_stream)
            for p, st in zip(parts, streams):
                p.synchronize(st)
            want = dict(full.outputs())
            if base_color:
                want["IN_MV"] = full.tex["IN_MV"]
                # (frame 0 clears IN_MV: from frame 1 on, a difference is the patch)
                patched |= f > 0 and not torch.equal(full.tex["IN_MV"].view(torch.int16), fr["IN_MV"].to(full.device).view(torch.int16))
            for name, t in want.items():
                got = torch.empty_like(t)
                for p, st in zip(parts, streams):
                    _copy_rows(p, name, got, False, st)
                torch.cuda.synchronize()
                same = got.view(torch.uint8) == t.view(torch.uint8)
                assert bool(same.all()), (f, schedule(f), name, float(same.float().mean()))
        assert patched or not base_color, "temporal stabilization never rewrote IN_MV: the IN_MV comparison proves nothing"
    finally:
        for p in parts:
            p.destroy()
        full.destroy()


@pytest.mark.parametrize("denoiser,world,halo,schedule,whole_frame_call,base_color", [
    ("REBLUR_DIFFUSE_SPECULAR", 2, 32, "constant", True, False),
    ("REBLUR_DIFFUSE_SPECULAR", 3, 96, "shrink_grow", False, False),
    ("REBLUR_DIFFUSE_SPECULAR", 4, 16, "first_strip_only", True, False),
    ("REBLUR_DIFFUSE_SPECULAR", 2, 16, "origin", True, False),
    ("REBLUR_DIFFUSE_SPECULAR", 3, 32, "origin", False, False),
    ("REBLUR_DIFFUSE_SPECULAR", 4, 16, "moving_origin", True, False),
    ("REBLUR_DIFFUSE_SPECULAR", 2, 16, "origin", True, True),
    ("REBLUR_DIFFUSE_SPECULAR", 3, 32, "moving_origin", False, True),
    ("RELAX_DIFFUSE_SPECULAR", 2, 16, "shrink_grow", True, False),
    ("RELAX_DIFFUSE_SPECULAR", 3, 32, "origin", False, False),
    ("RELAX_DIFFUSE_SPECULAR", 4, 16, "first_strip_only", True, False),
    ("SIGMA_SHADOW", 3, 16, "origin", True, False),
    ("SIGMA_SHADOW", 4, 96, "first_strip_only", False, False),
    ("SIGMA_SHADOW", 2, 32, "moving_origin", True, False),
    ("REFERENCE", 2, 16, "moving_origin", True, False),
    ("REFERENCE", 4, 32, "shrink_grow", False, False),
])
def test_dynamic_resolution_strips_bit_identical_to_full_frame(denoiser, world, halo, schedule, whole_frame_call, base_color):
    _run(denoiser, world, halo, schedule, whole_frame_call, base_color=base_color)


def test_dynamic_resolution_cost_balanced_strips_bit_identical_to_full_frame():
    _run("REBLUR_DIFFUSE_SPECULAR", 3, 32, "moving_origin", True, weighted=True)


def test_rect_origin_change_after_the_frame_start_is_refused():
    """Connected strips stage the guide inputs for the rectOrigin of the frame start (nrdCudaBarrier / nrdCudaDenoise): a dispatch
    of a frame whose CommonSettings moved the origin afterwards fails instead of reading inputs staged for another origin."""
    import torch
    from raytracingdenoiser_b200 import harness, nrd, scene, strips
    den = nrd.Denoiser.SIGMA_SHADOW
    parts = [strips.StripDenoiser(den, W, H, r, 2, halo_rows=16) for r in range(2)]
    try:
        for p in parts:
            p.connect_local(parts)
        streams = [torch.cuda.Stream() for _ in parts]
        fr = scene.Scene(200, 120).frame(0, "reblur")
        common = dict(resourceSize=(W, H), resourceSizePrev=(W, H), rectOrigin=(8, 40))
        for p, st in zip(parts, streams):
            p.dispatches(harness.make_common_settings(fr, 200, 120, 0, common=common))
            p.ctx.barrier(st.cuda_stream)
        moved = dict(common, rectOrigin=(8, 24))
        raw, _ = parts[0].dispatches(harness.make_common_settings(fr, 200, 120, 1, common=moved))
        with pytest.raises(nrd.NrdError):  # refused before anything is enqueued: the ranks stay in step
            parts[0].ctx.execute_raw(C.byref(raw[0]), streams[0].cuda_stream)
        for p, st in zip(parts, streams):
            p.synchronize(st)
    finally:
        for p in parts:
            p.destroy()
