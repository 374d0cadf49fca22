"""Re-cutting connected strips between frames (nrdCudaRepartition), on the multi-GPU data path run as contexts of ONE process on one
GPU (arenas connected by pointer, as in test_gpu_strips.py).  Every texture keeps its contents across a re-cut, so after every frame
every output -- and IN_MV, which REBLUR temporal stabilization patches when isBaseColorMetalnessAvailable is set -- must be
bit-identical to one full-frame context running the strip build of the kernels, which is never re-cut."""
import ctypes as C

import pytest

pytestmark = pytest.mark.gpu

W, H = 320, 192
TILES = H // 16
FULL = (0, 0, W, H)


def _min_rows(halo):
    return max(16, (halo + 15) // 16 * 16)


def _capacity(world):
    return H - 16 * (world - 1)  # room for the most uneven cut: every other rank keeps one tile row


def _cut(world, halo, cost):
    from raytracingdenoiser_b200 import strips
    _, cut = strips.partition_rows_weighted(H, world, cost, min_rows=_min_rows(halo), max_rows=_capacity(world))
    return cut


def _policy(world, halo, rects):
    """The policy of strips.StripDenoiser: a cut of the live rows, tiles(max(rectSize.y, rectSizePrev.y)), before every frame on
    which they change."""
    cuts, last = [], None
    for f, rect in enumerate(rects):
        live = (max(rect[3], rects[f - 1][3] if f else rect[3]) + 15) // 16
        cuts.append(_cut(world, halo, [1.0 if t < live else 0.0 for t in range(TILES)]) if last is not None and live != last else None)
        last = live
    return cuts


def _squeeze(world):
    """Every rank but the last keeps one tile row at the top: ranks 1 .. world-2 move to rows they never held (halo 16)."""
    return [(16 * r, 16 * (r + 1)) for r in range(world - 1)] + [(16 * (world - 1), H)]


def _schedule(name, world, halo):
    """[(rect (ox, oy, w, h), restart, cut before the frame or None)] per frame."""
    flat = [1.0] * TILES
    if name == "shrink_grow":  # into the first strip and back, re-cut at every change of the live rows
        rects = [FULL, FULL, (0, 0, 200, 40), (0, 0, 200, 40), (0, 0, 250, 100), FULL, FULL]
        return [(r, False, c) for r, c in zip(rects, _policy(world, halo, rects))]
    if name == "origin":  # rectOrigin.y != 0 across the re-cuts: the staged copies move too
        rects = [(24, 37, 250, 141), (24, 37, 250, 141), (24, 37, 160, 100), (16, 8, 160, 100), (8, 50, 250, 60), (8, 50, 250, 60)]
        return [(r, False, c) for r, c in zip(rects, _policy(world, halo, rects))]
    if name == "restart":  # a history reset right after a re-cut: the specular taps reach far past the ghost rows
        rects = [FULL, FULL, (0, 0, 250, 141), (0, 0, 250, 141), (0, 0, 250, 100), (0, 0, 250, 100)]
        return [(r, f == 3, c) for f, (r, c) in enumerate(zip(rects, _policy(world, halo, rects)))]
    if name == "never_held":  # no rect change; boundaries move by more than the halo, into rows a rank never held
        return [(FULL, False, None), (FULL, False, None), (FULL, False, _squeeze(world)), (FULL, False, None), (FULL, False, _cut(world, halo, flat))]
    if name == "many":  # re-cuts in a row, and back to the first partition
        top = _cut(world, halo, [8.0] * 3 + [1.0] * (TILES - 3))
        bottom = _cut(world, halo, [1.0] * (TILES - 3) + [8.0] * 3)
        return [(FULL, False, None), (FULL, False, top), (FULL, False, bottom), ((0, 0, 250, 141), False, top), ((0, 0, 250, 141), False, _cut(world, halo, flat))]
    raise KeyError(name)


def _placed_frame(scenes, mode, f, rect, prev):
    """(frame of resource-sized tensors, CommonSettings overrides) of frame f; scenes caches one scene per rect size."""
    import torch
    from raytracingdenoiser_b200 import harness, scene
    ox, oy, rw, rh = rect
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
    return placed, dict(resourceSize=(W, H), resourceSizePrev=(W, H), rectSizePrev=(prev[2], prev[3]), rectOrigin=(ox, oy))


def _copy_rows(part, name, tensor, to_context, stream):
    from raytracingdenoiser_b200 import nrd
    t = tensor[part.y0:part.y1]
    part.ctx.copy(getattr(nrd.ResourceType, name), 0, t.data_ptr(), t.stride(0) * t.element_size(), to_context, stream.cuda_stream)


def _check_rows(parts, den):
    """nrdCudaGetTexture: every rank reports its new rows, for user textures and (downsampled or not) pool textures."""
    from raytracingdenoiser_b200 import nrd
    pools = parts[0].instance.get_instance_desc()
    for p in parts:
        info = p.ctx.get_texture(nrd.ResourceType.IN_VIEWZ)
        assert (info.firstRow, info.firstRow + info.rowsNum) == (p.y0, p.y1)
        for kind, lst in ((nrd.ResourceType.PERMANENT_POOL, pools["permanentPool"]), (nrd.ResourceType.TRANSIENT_POOL, pools["transientPool"])):
            for i, (_, ds) in enumerate(lst):
                info = p.ctx.get_texture(kind, i)
                assert (info.firstRow, info.firstRow + info.rowsNum) == (p.y0 // ds, min((p.y1 + ds - 1) // ds, (H + ds - 1) // ds)), (den, kind, i, ds)


class _Rig(object):
    """One full-frame reference context and `world` connected strip contexts of this process."""

    def __init__(self, denoiser_name, world, halo, first_cut=None, capacity=None, base_color=False):
        import torch
        from raytracingdenoiser_b200 import harness, nrd, strips
        self.den = getattr(nrd.Denoiser, denoiser_name)
        self.mode = harness.radiance_mode(self.den)
        self.flags = {"isBaseColorMetalnessAvailable": True} if base_color else {}
        settings = None
        if base_color:  # thresholds low enough that the motion-vector patch rewrites part of IN_MV (as in test_gpu_reblur.py)
            settings = nrd.ReblurSettings()
            settings.specularProbabilityThresholdsForMvModification[0], settings.specularProbabilityThresholdsForMvModification[1] = 0.2, 0.6
        self.parts = []
        self.full = harness.GpuDenoiser(self.den, W, H, settings=settings, common=self.flags)
        capacity = capacity or _capacity(world)
        cut = first_cut or _cut(world, halo, [1.0] * TILES)
        self.parts = [strips.StripDenoiser(self.den, W, H, r, world, halo_rows=halo, partition=(capacity, cut), settings=settings) for r in range(world)]
        self.names = harness.denoiser_resources(self.den, self.flags)
        for p in self.parts:
            p.connect_local(self.parts)
        self.streams = [torch.cuda.Stream() for _ in self.parts]
        self.scenes = {}
        self.patched = False

    def repartition(self, cut):
        for p, st in zip(self.parts, self.streams):
            p.repartition(cut, st)

    def frame(self, f, rect, prev, restart=False, whole_frame_call=True, before_frame_start=None):
        import torch
        from raytracingdenoiser_b200 import harness, nrd
        fr, common = _placed_frame(self.scenes, self.mode, f, rect, prev)
        common.update(self.flags)
        if restart:
            common["accumulationMode"] = int(nrd.AccumulationMode.RESTART)
        cs = harness.make_common_settings(fr, rect[2], rect[3], f, common=common)
        self.full.set_inputs(fr)
        self.full.denoise(cs)
        torch.cuda.synchronize()
        for p, st in zip(self.parts, self.streams):
            for name in self.names:
                if name.startswith("IN_"):
                    _copy_rows(p, name, fr[name], True, st)
        if whole_frame_call:
            for p, st in zip(self.parts, self.streams):
                p.denoise(cs, st)
        else:
            # the application-driven path: SetCommonSettings, nrdCudaBarrier, the dispatch list, ranks interleaved pass by pass
            lists = [p.dispatches(cs) for p in self.parts]
            if before_frame_start:
                before_frame_start(lists)
            for p, st in zip(self.parts, self.streams):
                p.ctx.barrier(st.cuda_stream)
            n = lists[0][1]
            assert all(m == n for _, m in lists)
            for i in range(n):
                for p, st, (raw, _) in zip(self.parts, self.streams, lists):
                    p.ctx.execute_raw(C.byref(raw[i]), st.cuda_stream)
        for p, st in zip(self.parts, self.streams):
            p.synchronize(st)
        want = dict(self.full.outputs())
        if self.flags:
            want["IN_MV"] = self.full.tex["IN_MV"]
            self.patched |= f > 0 and not torch.equal(self.full.tex["IN_MV"].view(torch.int16), fr["IN_MV"].to(self.full.device).view(torch.int16))
        for name, t in want.items():
            got = torch.empty_like(t)
            for p, st in zip(self.parts, self.streams):
                _copy_rows(p, name, got, False, st)
            torch.cuda.synchronize()
            same = got.view(torch.uint8) == t.view(torch.uint8)
            assert bool(same.all()), (f, rect, [(p.y0, p.y1) for p in self.parts], name, float(same.float().mean()))

    def destroy(self):
        for p in self.parts:
            p.destroy()
        self.full.destroy()


def _run(denoiser_name, world, halo, schedule, whole_frame_call, base_color=False):
    import os
    os.environ["NRD_B200_FORCE_STRIP_KERNELS"] = "1"  # the full-frame reference runs the strip build of the kernels
    rig = None
    try:
        rig = _Rig(denoiser_name, world, halo, base_color=base_color)
        frames = _schedule(schedule, world, halo)
        cuts = 0
        for f, (rect, restart, cut) in enumerate(frames):
            if cut is not None:
                rig.repartition(cut)
                _check_rows(rig.parts, rig.den)
                cuts += 1
            rig.frame(f, rect, frames[f - 1][0] if f else rect, restart, whole_frame_call)
        assert cuts >= 2, frames
        assert rig.patched or not base_color, "temporal stabilization never rewrote IN_MV: the IN_MV comparison proves nothing"
    finally:  # a failing case must not leak its strip-mode contexts (there are only kMaxPeerSlots per process)
        if rig is not None:
            rig.destroy()
        del os.environ["NRD_B200_FORCE_STRIP_KERNELS"]


@pytest.mark.parametrize("denoiser,world,halo,schedule,whole_frame_call,base_color", [
    # (REBLUR with a halo that holds the whole other strip: with a smaller one, a growing rect hits the gap of
    # test_gpu_strips_rect_growth.py, which needs no re-cut)
    ("REBLUR_DIFFUSE_SPECULAR", 2, 96, "shrink_grow", True, False),
    ("REBLUR_DIFFUSE_SPECULAR", 2, 96, "shrink_grow", False, True),
    ("REBLUR_DIFFUSE_SPECULAR", 4, 16, "never_held", True, False),
    ("REBLUR_DIFFUSE_SPECULAR", 3, 16, "never_held", False, False),
    ("REBLUR_DIFFUSE_SPECULAR", 2, 96, "restart", True, False),
    ("REBLUR_DIFFUSE_SPECULAR", 4, 32, "restart", False, False),
    ("REBLUR_DIFFUSE_SPECULAR", 3, 16, "origin", False, True),
    ("REBLUR_DIFFUSE_SPECULAR", 4, 16, "many", True, False),
    ("RELAX_DIFFUSE_SPECULAR", 2, 32, "shrink_grow", False, False),
    ("RELAX_DIFFUSE_SPECULAR", 4, 16, "shrink_grow", True, False),
    ("RELAX_DIFFUSE_SPECULAR", 4, 16, "never_held", True, False),
    ("RELAX_DIFFUSE_SPECULAR", 3, 16, "restart", True, False),
    ("RELAX_DIFFUSE_SPECULAR", 2, 96, "many", False, False),
    ("SIGMA_SHADOW", 3, 16, "shrink_grow", True, False),
    ("SIGMA_SHADOW", 2, 32, "shrink_grow", False, False),
    ("SIGMA_SHADOW", 4, 16, "never_held", False, False),
    ("SIGMA_SHADOW", 2, 96, "origin", True, False),
    ("REFERENCE", 4, 32, "shrink_grow", False, False),
    ("REFERENCE", 2, 16, "shrink_grow", True, False),
    ("REFERENCE", 2, 16, "origin", True, False),
    ("REFERENCE", 3, 16, "many", True, False),
])
def test_repartition_bit_identical_to_full_frame(denoiser, world, halo, schedule, whole_frame_call, base_color):
    _run(denoiser, world, halo, schedule, whole_frame_call, base_color=base_color)


def test_refused_tables_enqueue_nothing():
    """Each refusal returns INVALID_ARGUMENT on every rank before anything is enqueued: the ranks stay in step and the next frames
    still match bit for bit.  Then a dispatch after a re-cut but before the next frame start is refused too."""
    import os
    from raytracingdenoiser_b200 import nrd
    os.environ["NRD_B200_FORCE_STRIP_KERNELS"] = "1"
    rig = None
    try:
        # 3 strips of 64 rows, 128 reserved, halo 32
        rig = _Rig("REBLUR_DIFFUSE_SPECULAR", 3, 32, first_cut=[(0, 64), (64, 128), (128, 192)], capacity=128)
        rig.frame(0, FULL, FULL)
        bad = {
            "does not cover the frame": [0, 64, 128, 176],
            "not a multiple of 16": [0, 64, 120, 192],
            "taller than stripHeight": [0, 144, 176, 192],
            "shorter than the halo": [0, 16, 64, 192],
            "a strip without rows": [0, 64, 64, 192],
        }
        for why, starts in bad.items():
            for p, st in zip(rig.parts, rig.streams):
                with pytest.raises(nrd.NrdError) as e:
                    p.ctx.repartition(starts, st.cuda_stream)
                assert e.value.result == nrd.Result.INVALID_ARGUMENT, why
            for p in rig.parts:
                info = p.ctx.get_texture(nrd.ResourceType.IN_VIEWZ)
                assert (info.firstRow, info.firstRow + info.rowsNum) == (p.y0, p.y1), why
        rig.frame(1, FULL, FULL)
        rig.repartition([(0, 96), (96, 128), (128, 192)])

        def dispatch_too_early(lists):
            raw, n = lists[0]
            for i in (0, n - 1):  # the first pass (it builds the guide) and the last: both need a frame start first
                with pytest.raises(nrd.NrdError) as e:
                    rig.parts[0].ctx.execute_raw(C.byref(raw[i]), rig.streams[0].cuda_stream)
                assert e.value.result == nrd.Result.FAILURE
        rig.frame(2, FULL, FULL, whole_frame_call=False, before_frame_start=dispatch_too_early)
        rig.frame(3, FULL, FULL)
    finally:
        if rig is not None:
            rig.destroy()
        del os.environ["NRD_B200_FORCE_STRIP_KERNELS"]


def test_repartition_needs_connected_strips():
    """UNSUPPORTED on a one-GPU context and on a strip context that is not connected; a connected world of one accepts the identity
    table only, and does nothing."""
    from raytracingdenoiser_b200 import nrd, strips
    inst = nrd.Instance([(0, nrd.Denoiser.SIGMA_SHADOW)])
    one = nrd.CudaContext(inst, W, H)
    lone = strips.StripDenoiser(nrd.Denoiser.SIGMA_SHADOW, W, H, 0, 2, halo_rows=16)
    single = strips.StripDenoiser(nrd.Denoiser.SIGMA_SHADOW, W, H, 0, 1, halo_rows=16)
    try:
        for ctx in (one, lone.ctx):
            with pytest.raises(nrd.NrdError) as e:
                ctx.repartition([0, 96, H])
            assert e.value.result == nrd.Result.UNSUPPORTED
        single.connect_local([single])
        single.repartition([(0, H)])
        with pytest.raises(nrd.NrdError) as e:
            single.ctx.repartition([0, H - 16])
        assert e.value.result == nrd.Result.INVALID_ARGUMENT
        info = single.ctx.get_texture(nrd.ResourceType.IN_VIEWZ)
        assert (info.firstRow, info.rowsNum) == (0, H)
    finally:
        single.destroy()
        lone.destroy()
        one.destroy()
        inst.destroy()
