"""GPU parity of the auxiliary passes against the oracle: split-screen passes of the three families (CommonSettings::splitScreen)
and the REFERENCE denoiser."""
import json
import os

import pytest

pytestmark = pytest.mark.gpu


def _dump(name, report):
    out = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "gpurun_out")
    os.makedirs(out, exist_ok=True)
    with open(os.path.join(out, name), "w") as f:
        json.dump(report, f, indent=1)


@pytest.mark.parametrize("denoiser_name,split", [
    ("REBLUR_DIFFUSE_SPECULAR", 0.4), ("REBLUR_SPECULAR", 1.0), ("RELAX_DIFFUSE_SPECULAR", 0.4), ("RELAX_DIFFUSE", 0.6),
    ("SIGMA_SHADOW", 0.5), ("SIGMA_SHADOW_TRANSLUCENCY", 0.5),
])
def test_split_screen_per_pass(denoiser_name, split):
    """splitScreen in (0, 1): the whole chain plus the split-screen pass; splitScreen >= 1: the split-screen pass alone
    (Source/Reblur.cpp:120-128, Relax.cpp:196-204, Sigma.cpp:38-46)."""
    import parity
    from raytracingdenoiser_b200 import nrd
    sbs = parity.SideBySide(getattr(nrd.Denoiser, denoiser_name), 250, 141, common={"splitScreen": split})
    report = sbs.run_per_pass(3)
    shaders = [r["shader"] for r in report]
    assert any("SplitScreen" in s for s in shaders)
    if split >= 1.0:
        assert all("SplitScreen" in s or s.startswith("Clear_") for s in shaders), shaders
    _dump("parity_split_%s.json" % denoiser_name, report)
    assert not sbs.failures(), sbs.describe_failures()


def test_reference_denoiser_per_pass_and_sequence():
    """Denoiser::REFERENCE: running average of IN_SIGNAL in an RGBA32F history (Source/Denoisers/Reference.hpp)."""
    import numpy as np
    import parity
    from raytracingdenoiser_b200 import nrd
    sbs = parity.SideBySide(nrd.Denoiser.REFERENCE, 250, 141)
    report = sbs.run_per_pass(4)
    assert {r["shader"] for r in report} >= {"REFERENCE_TemporalAccumulation.cs", "REFERENCE_Copy.cs"}
    _dump("parity_REFERENCE.json", report)
    assert not sbs.failures(), sbs.describe_failures()
    res = parity.run_sequence(nrd.Denoiser.REFERENCE, 320, 180, 6)
    for name, (frac, psnr) in res.items():
        assert frac >= 0.999 and psnr >= 60.0, (name, frac, psnr)


def _rects(f):
    """Dynamic resolution: the rect changes size after two frames and sits at a non-zero origin of the G-buffer inputs."""
    return (16, 8, 250, 141) if f < 2 else (24, 16, 280, 158)


@pytest.mark.parametrize("denoiser_name", ["REBLUR_DIFFUSE_SPECULAR", "RELAX_DIFFUSE_SPECULAR", "SIGMA_SHADOW"])
def test_dynamic_resolution_per_pass(denoiser_name):
    """rectSize < resourceSize, rectOrigin != 0, rectSizePrev != rectSize (Source/InstanceImpl.cpp:834-856, Common.hlsli:200-222):
    textures are 320x192, the passes run over a 250x141 rect and then over a 280x158 one."""
    import parity
    from raytracingdenoiser_b200 import nrd
    sbs = parity.SideBySide(getattr(nrd.Denoiser, denoiser_name), 320, 192, noise_floor=denoiser_name.startswith("RELAX"))
    report = sbs.run_per_pass(4, rect_fn=_rects)
    _dump("parity_dynres_%s.json" % denoiser_name, report)
    assert not sbs.failures(), sbs.describe_failures()


def test_user_textures_in_wider_formats_give_the_same_result():
    """Include/NRDDescs.h lists MINIMUM formats: a user texture may be bound in a wider float format (RGBA32_SFLOAT radiance / motion /
    outputs, R16_SFLOAT viewZ whose values fit).  The executor converts around the passes; with inputs that convert exactly, the
    outputs must equal those of a run with the kernels' own formats, bit for bit."""
    import torch
    from raytracingdenoiser_b200 import harness, nrd, scene
    w, h, frames = 250, 141, 4
    den = nrd.Denoiser.REBLUR_DIFFUSE_SPECULAR
    sc = scene.Scene(w, h)
    frs = []
    for f in range(frames):
        fr = sc.frame(f)
        fr["IN_VIEWZ"] = fr["IN_VIEWZ"].to(torch.float16).to(torch.float32)  # values a R16_SFLOAT texture can hold
        frs.append(fr)
    native = harness.GpuDenoiser(den, w, h)
    for f, fr in enumerate(frs):
        native.set_inputs(fr)
        native.denoise(harness.make_common_settings(fr, w, h, f))
    torch.cuda.synchronize()
    want = {k: v.clone() for k, v in native.outputs().items()}
    native.destroy()

    inst = nrd.Instance([(0, den)])
    ctx = nrd.CudaContext(inst, w, h)
    dev = torch.device("cuda", 0)
    wide = {"IN_MV": (nrd.Format.RGBA32_SFLOAT, torch.float32, 4), "IN_VIEWZ": (nrd.Format.R16_SFLOAT, torch.float16, 1),
            "IN_DIFF_RADIANCE_HITDIST": (nrd.Format.RGBA32_SFLOAT, torch.float32, 4), "IN_SPEC_RADIANCE_HITDIST": (nrd.Format.RGBA16_SFLOAT, torch.float16, 4),
            "OUT_DIFF_RADIANCE_HITDIST": (nrd.Format.RGBA32_SFLOAT, torch.float32, 4), "OUT_SPEC_RADIANCE_HITDIST": (nrd.Format.RGBA32_SFLOAT, torch.float32, 4),
            "IN_NORMAL_ROUGHNESS": harness.USER_FORMATS["IN_NORMAL_ROUGHNESS"]}
    tex = {}
    for name, (fmt, dtype, ch) in wide.items():
        t = torch.zeros((h, w, ch) if ch > 1 else (h, w), dtype=dtype, device=dev)
        tex[name] = t
        ctx.set_user_texture(getattr(nrd.ResourceType, name), t.data_ptr(), t.stride(0) * t.element_size(), fmt)
    with pytest.raises(nrd.NrdError):  # fewer channels / lower precision than the minimum is refused
        bad = torch.zeros((h, w), dtype=torch.float16, device=dev)
        ctx.set_user_texture(nrd.ResourceType.IN_DIFF_RADIANCE_HITDIST, bad.data_ptr(), bad.stride(0) * 2, nrd.Format.R16_SFLOAT)
    ctx.set_user_texture(nrd.ResourceType.IN_DIFF_RADIANCE_HITDIST, tex["IN_DIFF_RADIANCE_HITDIST"].data_ptr(), tex["IN_DIFF_RADIANCE_HITDIST"].stride(0) * 4, nrd.Format.RGBA32_SFLOAT)
    for f, fr in enumerate(frs):
        for name, t in tex.items():
            if name.startswith("IN_"):
                src = fr[name].to(dev)
                t.copy_(src.to(t.dtype) if t.dtype != src.dtype and t.dtype.is_floating_point else src)
        inst.set_common_settings(harness.make_common_settings(fr, w, h, f))
        ctx.denoise([0], stream=torch.cuda.current_stream(dev).cuda_stream)
    torch.cuda.synchronize()
    for name in ("OUT_DIFF_RADIANCE_HITDIST", "OUT_SPEC_RADIANCE_HITDIST"):
        got = tex[name]
        assert got.abs().sum().item() > 0
        assert torch.equal(got, want[name].to(torch.float32)), name
    ctx.destroy()
    inst.destroy()


@pytest.mark.parametrize("denoiser_name", ["REBLUR_DIFFUSE_SPECULAR", "SIGMA_SHADOW_TRANSLUCENCY"])
def test_user_textures_and_formats_match_the_python_table(denoiser_name):
    """The executor's user textures and their formats against harness.USER_FORMATS, which applications and bench.py read:
    binding a user texture in its listed format succeeds exactly for the listed types (others are UNSUPPORTED), and a strip-mode
    context that covers the whole frame holds exactly the listed textures, in that format."""
    import torch
    from raytracingdenoiser_b200 import harness, nrd
    den = getattr(nrd.Denoiser, denoiser_name)
    w, h = 64, 32
    inst = nrd.Instance([(0, den)])
    ctx = nrd.CudaContext(inst, w, h)
    strip = nrd.CudaContext(inst, w, h, strip=(0, h), strip_height=h)
    texels = torch.zeros((h, w, 16), dtype=torch.uint8, device="cuda")  # 16 bytes per texel: room for every format
    try:
        for rt in nrd.ResourceType:
            if rt >= nrd.ResourceType.TRANSIENT_POOL:
                continue
            listed = rt.name in harness.USER_FORMATS
            fmt = harness.user_format(den, rt.name)[0] if listed else nrd.Format.RGBA32_SFLOAT
            if listed:
                ctx.set_user_texture(rt, texels.data_ptr(), texels.stride(0), fmt)
                info = strip.get_texture(rt)
                assert (info.format, info.width, info.height, info.firstRow, info.rowsNum) == (int(fmt), w, h, 0, h), rt.name
            else:
                with pytest.raises(nrd.NrdError) as e:
                    ctx.set_user_texture(rt, texels.data_ptr(), texels.stride(0), fmt)
                assert e.value.result == nrd.Result.UNSUPPORTED, rt.name
                with pytest.raises(nrd.NrdError):
                    strip.get_texture(rt)
    finally:
        strip.destroy()
        ctx.destroy()
        inst.destroy()
