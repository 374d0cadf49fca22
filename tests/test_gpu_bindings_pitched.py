"""User textures bound as pitched views into larger allocations (nrdCudaSetUserTexture takes any pitch).

Every user texture, input and output, is a view into an allocation with guard rows above and below and guard columns to the right
of the view, filled with NaN bit patterns (float formats) or 0xA5 bytes (the others).  Two layouts:
  padded:    pitch = width * bytes per texel rounded up to 256 B, plus 256 B; the base is 256-byte aligned
  unaligned: pitch = (width + 3) * bytes per texel and the base one texel past the start of a row, so that the base is not
             16-byte aligned (nor, mostly, the pitch): the executor and the kernels cannot stage such a surface with TMA, and clears
             of it cannot use the aligned path
The outputs must be bit-identical to a run with contiguous bindings, no guard byte may change, and no input may be written.  One
input is written by design, as in the reference: IN_MV (the frame-0 clear zeroes it; REBLUR temporal stabilization with
isBaseColorMetalnessAvailable replaces the motion of specular-dominant pixels).  IN_MV is therefore compared with IN_MV of the
contiguous run after every frame instead of with what was uploaded."""
import pytest

pytestmark = pytest.mark.gpu

GUARD_ROWS = 2
ALL_OPTIONAL_INPUTS = {"isHistoryConfidenceAvailable": True, "isDisocclusionThresholdMixAvailable": True, "isBaseColorMetalnessAvailable": True}


class PitchedView(object):
    """A (height, width[, channels]) view with a foreign pitch into a guard-filled allocation."""

    def __init__(self, width, height, channels, dtype, layout, device):
        import torch
        esize = torch.empty((), dtype=dtype).element_size()
        bpt = esize * channels
        if layout == "padded":
            self.pitch = (width * bpt + 255) // 256 * 256 + 256
            base = GUARD_ROWS * self.pitch
        else:
            self.pitch = (width + 3) * bpt
            base = GUARD_ROWS * self.pitch + bpt
        total = (base + (height + GUARD_ROWS) * self.pitch + 15) // 16 * 16
        self.raw = torch.empty(total, dtype=torch.uint8, device=device)
        if dtype == torch.float16:
            self.raw.view(torch.int16).fill_(0x7D5A)          # a NaN
        elif dtype == torch.float32:
            self.raw.view(torch.int32).fill_(0x7FA5A5A5)      # a NaN
        else:
            self.raw.fill_(0xA5)
        shape, strides = ((height, width, channels), (self.pitch // esize, channels, 1)) if channels > 1 else ((height, width), (self.pitch // esize, 1))
        self.view = self.raw.view(dtype).as_strided(shape, strides, base // esize)
        rows = base + torch.arange(height, device=device)[:, None] * self.pitch + torch.arange(width * bpt, device=device)[None, :]
        self.guard_mask = torch.ones(total, dtype=torch.bool, device=device)
        self.guard_mask[rows.reshape(-1)] = False
        self.guard = self.raw[self.guard_mask].clone()
        self.ptr = self.raw.data_ptr() + base
        assert layout == "padded" or self.ptr % 16 != 0

    def guard_intact(self):
        import torch
        return torch.equal(self.raw[self.guard_mask], self.guard)


def _bytes(t):
    import torch
    return t.contiguous().view(-1).view(torch.uint8)


def _frames(den, w, h, frames):
    from raytracingdenoiser_b200 import harness, scene
    sc = scene.Scene(w, h)
    return [sc.frame(f, harness.radiance_mode(den)) for f in range(frames)]


def _contiguous_run(den, w, h, frs, common):
    """Outputs and IN_MV after every frame of a run with harness.GpuDenoiser's contiguous bindings."""
    import torch
    from raytracingdenoiser_b200 import harness
    g = harness.GpuDenoiser(den, w, h, common=common)
    states = []
    for f, fr in enumerate(frs):
        g.set_inputs(fr)
        g.denoise(harness.make_common_settings(fr, w, h, f, common=common))
        torch.cuda.synchronize()
        states.append({k: v.clone() for k, v in g.tex.items() if k.startswith("OUT_") or k == "IN_MV"})
    g.destroy()
    return states


def _pitched_run(den, w, h, frs, common, layout, formats, want):
    import torch
    from raytracingdenoiser_b200 import harness, nrd
    dev = torch.device("cuda", 0)
    inst = nrd.Instance([(0, den)])
    ctx = nrd.CudaContext(inst, w, h)
    views = {}
    try:
        for name in harness.denoiser_resources(den, common):
            fmt, dtype, ch = formats.get(name, harness.user_format(den, name))
            views[name] = PitchedView(w, h, ch, dtype, layout, dev)
            ctx.set_user_texture(getattr(nrd.ResourceType, name), views[name].ptr, views[name].pitch, fmt)
        for f, fr in enumerate(frs):
            for name, v in views.items():
                if name.startswith("IN_"):
                    v.view.copy_(fr[name].to(dev).to(v.view.dtype))
            inst.set_common_settings(harness.make_common_settings(fr, w, h, f, common=common))
            ctx.denoise([0], stream=torch.cuda.current_stream(dev).cuda_stream)
            torch.cuda.synchronize()
            for name, v in views.items():
                assert v.guard_intact(), "frame %d: a guard byte around %s changed" % (f, name)
                if name.startswith("OUT_") or (name == "IN_MV" and name not in formats):
                    ref = want[f][name].to(v.view.dtype)
                    assert torch.equal(_bytes(v.view), _bytes(ref)), "frame %d: %s differs from the contiguous run" % (f, name)
                else:
                    assert torch.equal(_bytes(v.view), _bytes(fr[name].to(dev).to(v.view.dtype))), "frame %d: input %s was written" % (f, name)
            assert any(float(v.view.float().abs().sum()) > 0 for k, v in views.items() if k.startswith("OUT_"))
    finally:
        ctx.destroy()
        inst.destroy()


CASES = [("REBLUR_DIFFUSE_SPECULAR", ALL_OPTIONAL_INPUTS), ("RELAX_DIFFUSE_SPECULAR", ALL_OPTIONAL_INPUTS),
         ("SIGMA_SHADOW_TRANSLUCENCY", None), ("REFERENCE", None)]


@pytest.mark.parametrize("layout", ["padded", "unaligned"])
@pytest.mark.parametrize("width,height", [(250, 141), (17, 17)])
@pytest.mark.parametrize("denoiser_name,common", CASES, ids=[c[0] for c in CASES])
def test_pitched_user_textures_give_the_contiguous_result(denoiser_name, common, width, height, layout):
    from raytracingdenoiser_b200 import nrd
    den = getattr(nrd.Denoiser, denoiser_name)
    frs = _frames(den, width, height, 4)
    want = _contiguous_run(den, width, height, frs, common)
    _pitched_run(den, width, height, frs, common, layout, {}, want)


def test_pitched_user_textures_in_a_wider_format():
    """IN_MV, the radiance inputs and the outputs as RGBA32_SFLOAT views with a padded pitch: the executor converts them around the
    passes (ConvertFormatKernel) reading and writing with the user's pitch.  fp16 inputs convert exactly, so the outputs equal the
    fp16 outputs of the contiguous run, widened.  An input in a wider format is converted into the kernels' copy and never
    converted back, so the frame-0 clear of IN_MV only zeroes that copy: the application's IN_MV must stay as uploaded."""
    import torch
    from raytracingdenoiser_b200 import nrd
    den, w, h = nrd.Denoiser.REBLUR_DIFFUSE_SPECULAR, 250, 141
    wide = (nrd.Format.RGBA32_SFLOAT, torch.float32, 4)
    formats = {k: wide for k in ("IN_MV", "IN_DIFF_RADIANCE_HITDIST", "IN_SPEC_RADIANCE_HITDIST", "OUT_DIFF_RADIANCE_HITDIST", "OUT_SPEC_RADIANCE_HITDIST")}
    frs = _frames(den, w, h, 4)
    want = _contiguous_run(den, w, h, frs, None)
    _pitched_run(den, w, h, frs, None, "padded", formats, want)
