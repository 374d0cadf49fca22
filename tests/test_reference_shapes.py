"""The CPU side of the small-frame GPU tests (tests/test_gpu_shapes.py) pinned at the same kind of sizes.

The GPU tests hold the kernels to the oracle at frames smaller than a CTA, a tile or a stencil.  That only means something if the
oracle, and the dispatch stream both run from, are right at those sizes too:
  * the product scheduler must emit the reference host code's dispatch stream (grids, downsampled pool sizes, constants) at
    1x1, 7x5, 17x17, 33x9 and 9x130;
  * the oracle's passes must equal the reference's own shaders at 17x9 and 33x130, with the per-shader gates of
    test_reference_shaders.test_oracle_pass_equals_the_reference_shader;
  * the parity harness must measure the noise floor of the dynamic-resolution loop on the same state as the oracle."""
import os

import numpy as np
import pytest

import test_reference_scheduler as rsched
import test_reference_shaders as rshaders
from raytracingdenoiser_b200 import nrd, scene

SCHEDULER_SIZES = [(1, 1), (7, 5), (17, 17), (33, 9), (9, 130)]
SHADER_SIZES = [(17, 9), (33, 130)]


def _dynres_fits(w, h):
    """The "dynres" camera of test_reference_scheduler renders a rect of 3/4 x 2/3 of the resource: it needs a rect of one texel."""
    return w * 3 // 4 >= 1 and h * 2 // 3 >= 1


@pytest.mark.skipif(not os.path.exists(rsched.REF_LIB), reason="oracle/_ref/libnrd_ref.so is built by build() from the reference")
@pytest.mark.parametrize("width,height", SCHEDULER_SIZES, ids=["%dx%d" % s for s in SCHEDULER_SIZES])
@pytest.mark.parametrize("denoiser_name", rsched.SUPPORTED)
def test_dispatch_stream_identical_to_reference_host_code_at_small_sizes(denoiser_name, width, height):
    ref_lib = rsched._ref_lib()
    den = getattr(nrd.Denoiser, denoiser_name)
    variants = ["default"] + (["dynres"] if _dynres_fits(width, height) else [])
    for variant in variants:
        checked = rsched._compare_streams(ref_lib, den, None, variant, w=width, h=height)
        assert checked["dispatches"] > 0, (variant, checked)


def _binary_shadow_left_of_split(size):
    """True when the left half of every frame is fully lit or fully shadowed (IN_PENUMBRA holds only 0 and the no-occluder value)."""
    w, h = size
    sc = scene.Scene(w, h)
    for f in range(2):
        pen = sc.frame(f)["IN_PENUMBRA"].float().numpy()[:, : (w + 1) // 2]
        if not set(np.unique(pen).tolist()) <= {0.0, 65504.0}:
            return False
    return True


SHADER_CASES = [n for n in sorted(rshaders.CASES) if not n.endswith("_dynamic_resolution")]  # those have a fixed resource size


@pytest.mark.skipif(not rshaders._have_shaders(), reason="oracle/_ref/shaders is built from the reference")
@pytest.mark.parametrize("width,height", SHADER_SIZES, ids=["%dx%d" % s for s in SHADER_SIZES])
@pytest.mark.parametrize("name", SHADER_CASES)
def test_oracle_pass_equals_the_reference_shader_at_small_sizes(name, width, height):
    """Checkerboarded inputs need an even width (scene.checkerboard_frame): those cases run one column wider."""
    size = (width + 1, height) if "checkerboard" in name and width % 2 else (width, height)
    stats, missing = rshaders.run_case(name, size=size)
    assert stats, "no pass of this case has a compiled reference shader"
    assert all(m.startswith("Clear_") for m in missing), missing
    for shader, s in stats.items():
        if "Tiles" not in shader:  # (a static scene classifies its tiles the same way every frame)
            if shader.startswith("SIGMA_") and shader.endswith("_SplitScreen") and s["changed"] == 0.0:
                # the split-screen pass writes IsLit(penumbra) left of the split; at 17x9 that half is only lit or shadowed
                # texels, which the chain before it already outputs exactly, so it rewrites the same bytes
                assert _binary_shadow_left_of_split(size), (shader, s)
            else:
                assert s["changed"] > 0.0, (shader, "the reference shader wrote nothing")
        if name == "reblur_checkerboard" and shader.endswith("_PrePass"):
            # the exact tap ties of the module docstring of test_reference_shaders (frame 0, identity rotator, blur radius of
            # one pixel): at these sizes most pixels have the minimum radius, so up to a quarter of frame 0 lands on the other
            # neighbour; every later frame is bit-identical but for the one-texel tap of the 33x130 case below
            assert s["min_bytes_equal_after_frame0"] >= (0.9995 if height == 130 else 1.0), (shader, s)
        elif size == (33, 130) and shader.startswith("REBLUR") and any(k in shader for k in ("PrePass", "_Blur", "PostBlur")):
            # a tap within one rounding of a texel border (test_reblur_at_640x360_against_the_reference_shaders): one texel here
            assert s["min_fraction"] >= 0.9995, (shader, s)
        elif any(k in shader for k in rshaders.ROUNDING_SENSITIVE):
            assert s["min_fraction"] >= 0.997, (shader, s)
        else:
            assert s["min_bytes_equal"] == 1.0, (shader, s)


class _OracleFollowingTheRect(object):
    """The oracle in the role of the CUDA executor, reading the inputs at the rect origin the harness uses for the frame."""

    def __init__(self, sbs):
        import oracle_runner as orr
        self.sbs = sbs
        self.den = orr.CpuDenoiser(sbs.denoiser, sbs.w, sbs.h, identifier=sbs.identifier, instance=sbs.instance, common=sbs.common)

    def upload(self, rtype, index, arr):
        self.den.resolve(rtype, index)[0][...] = arr

    def download(self, rtype, index, out):
        out[...] = self.den.resolve(rtype, index)[0]

    def execute_raw(self, ref):
        self.den.rect_origin = self.sbs.cpu.rect_origin
        self.den.run_dispatch(nrd.Dispatch(ref._obj, self.sbs.instance.get_instance_desc()["pipelines"]))


def test_noise_floor_of_the_dynamic_resolution_loop_is_measured_on_the_oracle_state():
    """The "fma" and "uv" builds of the oracle run every floor pass of the rect loop on the inputs the oracle gets: their
    disagreement with it stays a rounding floor (a floor read from stale textures would be near 0 and pass anything)."""
    import parity
    rects = [(0, 0, 64, 48), (63, 47, 1, 1), (40, 30, 24, 18), (0, 0, 17, 9), (0, 0, 64, 48)]
    sbs = parity.SideBySide(nrd.Denoiser.RELAX_DIFFUSE_SPECULAR, 64, 48, noise_floor=True, floor_passes=("",), executor=_OracleFollowingTheRect)
    report = sbs.run_per_pass(5, rect_fn=lambda f: rects[f])
    assert {r["frame"] for r in report} == set(range(5))
    assert all("floor_fraction" in r for r in report)
    assert min(r["floor_fraction"] for r in report) >= 0.99, min(report, key=lambda r: r["floor_fraction"])
    assert not sbs.failures(), sbs.describe_failures()
