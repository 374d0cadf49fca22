"""Every launcher checks that a dispatch binds exactly the textures its pass reads: a DispatchDesc with one binding too many is
refused with Result::FAILURE, names the shader in nrdCudaGetLastError and launches nothing."""
import ctypes as C

import pytest

pytestmark = pytest.mark.gpu

W, H = 128, 72

# one pass of every family launcher: (denoiser, ReblurSettings / RelaxSettings overrides, CommonSettings overrides, shader)
CASES = [
    ("REBLUR_DIFFUSE_SPECULAR", {"hitDistanceReconstructionMode": "AREA_3X3"}, None, "REBLUR_DiffuseSpecular_HitDistReconstruction.cs"),
    ("REBLUR_DIFFUSE_SPECULAR", None, None, "REBLUR_DiffuseSpecular_TemporalAccumulation.cs"),
    ("REBLUR_DIFFUSE_SPECULAR", None, None, "REBLUR_DiffuseSpecular_Blur.cs"),
    ("RELAX_DIFFUSE", None, None, "RELAX_Diffuse_TemporalAccumulation.cs"),
    ("SIGMA_SHADOW", None, None, "SIGMA_Shadow_Blur.cs"),
    ("REBLUR_SPECULAR", None, {"splitScreen": 1.0}, "REBLUR_Specular_SplitScreen.cs"),
    ("REFERENCE", None, None, "REFERENCE_Copy.cs"),
]


def _with_extra_binding(raw):
    """A copy of the DispatchDesc whose last binding is bound a second time."""
    from raytracingdenoiser_b200 import nrd
    n = raw.resourcesNum
    resources = (nrd.ResourceDesc * (n + 1))()
    for k in range(n):
        resources[k] = raw.resources[k]
    resources[n] = raw.resources[n - 1]
    bad = nrd.DispatchDesc.from_buffer_copy(raw)
    bad.resources = C.cast(resources, C.POINTER(nrd.ResourceDesc))
    bad.resourcesNum = n + 1
    return bad, resources


@pytest.mark.parametrize("denoiser_name,settings,common,shader", CASES, ids=[c[3] for c in CASES])
def test_extra_binding_is_refused(denoiser_name, settings, common, shader):
    import torch
    from raytracingdenoiser_b200 import harness, nrd, scene
    den = getattr(nrd.Denoiser, denoiser_name)
    s = None
    if settings:
        s = nrd.ReblurSettings() if denoiser_name.startswith("REBLUR") else nrd.RelaxSettings()
        s.hitDistanceReconstructionMode = int(getattr(nrd.HitDistanceReconstructionMode, settings["hitDistanceReconstructionMode"]))
    g = harness.GpuDenoiser(den, W, H, settings=s, common=common)
    fr = scene.Scene(W, H).frame(0, harness.radiance_mode(den))
    g.set_inputs(fr)
    g.instance.set_common_settings(harness.make_common_settings(fr, W, H, 0, common=common))
    r, raw, n = g.instance.get_compute_dispatches_raw([g.identifier])
    assert r == nrd.Result.SUCCESS
    pipelines = g.instance.get_instance_desc()["pipelines"]
    stream = torch.cuda.current_stream(g.device).cuda_stream
    found = False
    for i in range(n):
        if nrd.Dispatch(raw[i], pipelines).shaderFileName != shader:
            g.ctx.execute_raw(C.byref(raw[i]), stream)  # the passes before it, so that it runs on the state it expects
            continue
        found = True
        bad, _keep = _with_extra_binding(raw[i])
        launches = nrd.launch_count()
        with pytest.raises(nrd.NrdError) as refused:
            g.ctx.execute_raw(C.byref(bad), stream)
        assert refused.value.result == nrd.Result.FAILURE
        assert shader in str(refused.value)
        assert nrd.launch_count() == launches
        g.ctx.execute_raw(C.byref(raw[i]), stream)  # the dispatch as scheduled still runs
        assert nrd.launch_count() == launches + 1
        break
    torch.cuda.synchronize()
    g.destroy()
    assert found, shader
