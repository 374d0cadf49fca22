"""The second staging path of HistoryFix, TemporalStabilization and hit-distance reconstruction: clamped loads instead of TMA.

The kernels take it for a surface TMA cannot address (base or pitch not 16-byte aligned) or when NRD_B200_NO_TMA=1 is set.  Pool
textures always have 256-byte rows, so only the variable reaches it for them.  It is read once per process, so a child process
runs the frames with it set and stores every texture every dispatch wrote; this process runs the same frames with TMA and
demands the same bytes, dispatch by dispatch."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

FRAMES = 6
SIZES = [(250, 141), (7, 5)]
SETTINGS = ["default", "hitdist3x3", "hitdist5x5", "perf"]


def _settings(key):
    from raytracingdenoiser_b200 import nrd
    hd = nrd.HitDistanceReconstructionMode
    return {"default": None,
            "hitdist3x3": nrd.ReblurSettings(hitDistanceReconstructionMode=int(hd.AREA_3X3)),
            "hitdist5x5": nrd.ReblurSettings(hitDistanceReconstructionMode=int(hd.AREA_5X5)),
            "perf": nrd.ReblurSettings(enablePerformanceMode=True)}[key]


def record_dispatches(key, width, height):
    """{"f<frame>_d<dispatch>_<shader>_<resource>[<index>]": bytes of the texture} for every texture every dispatch writes."""
    import torch
    from raytracingdenoiser_b200 import harness, nrd, scene
    den = nrd.Denoiser.REBLUR_DIFFUSE_SPECULAR
    g = harness.GpuDenoiser(den, width, height, settings=_settings(key))
    sc = scene.Scene(width, height)
    stream = torch.cuda.current_stream(g.device).cuda_stream
    out = {}
    for f in range(FRAMES):
        fr = sc.frame(f, harness.radiance_mode(den))
        g.set_inputs(fr)
        g.instance.set_common_settings(harness.make_common_settings(fr, width, height, f))
        r, raw, n = g.instance.get_compute_dispatches_raw([g.identifier])
        assert r == nrd.Result.SUCCESS
        pipelines = g.instance.get_instance_desc()["pipelines"]
        for i in range(n):
            d = nrd.Dispatch(raw[i], pipelines)
            g.ctx.execute_raw(C.byref(raw[i]), stream)
            torch.cuda.synchronize()
            for dtype_, rtype, index in d.resources:
                if dtype_ != nrd.DescriptorType.STORAGE_TEXTURE:
                    continue
                info = g.ctx.get_texture(rtype, index)
                arr = np.empty((info.rowsNum, info.width * nrd.FORMAT_BYTES[nrd.Format(info.format)]), dtype=np.uint8)
                g.ctx.download(rtype, index, arr)
                out["f%d_d%02d_%s_%s[%d]" % (f, i, d.shaderFileName, nrd.ResourceType(rtype).name, index)] = arr
    g.destroy()
    return out


@pytest.mark.parametrize("width,height", SIZES)
@pytest.mark.parametrize("key", SETTINGS)
def test_clamped_load_staging_equals_tma_staging(key, width, height, tmp_path):
    assert "NRD_B200_NO_TMA" not in os.environ, "this process must run with TMA"
    path = str(tmp_path / "no_tma.npz")
    env = dict(os.environ, NRD_B200_NO_TMA="1")
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [os.path.abspath(__file__), key, str(width), str(height), path]
    child = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=600)
    assert child.returncode == 0, child.stdout[-2000:] + child.stderr[-4000:]
    want = record_dispatches(key, width, height)
    with np.load(path) as got:
        assert sorted(got.files) == sorted(want), "the two runs dispatched different passes"
        staged = [k for k in want if any(p in k for p in ("HistoryFix", "TemporalStabilization", "HitDistReconstruction"))]
        assert staged
        differ = [k for k in sorted(want) if not np.array_equal(got[k], want[k])]
    assert not differ, "NRD_B200_NO_TMA=1 changes %d of %d textures, first: %s" % (len(differ), len(want), differ[:8])


if __name__ == "__main__":  # the child: python test_gpu_no_tma.py <settings> <width> <height> <out.npz>
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path[:0] = [root]
    key_, w_, h_, out_ = sys.argv[1], int(sys.argv[2]), int(sys.argv[3]), sys.argv[4]
    np.savez(out_, **record_dispatches(key_, w_, h_))
