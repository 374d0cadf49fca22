"""GPU per-pass parity at the frame sizes and rects where index, clamp and staging code goes wrong.

The other parity tests run frames of 250x141 and more with the rect at the origin.  Here the frame is smaller than a CTA
(32x8, 32x4, 16x16), than a 16x16 classification tile, than the TMA boxes of HistoryFix (48x12) and TemporalStabilization
(36x10) and than the 5x5 hit-distance window, so that both frame edges fall inside one CTA, one stencil and one staged box:

  1x1, 1x64, 64x1   both edges inside every stencil and every CTA
  7x5, 40x3         smaller than the 5x5 window and the TMA halos
  16x16, 17x17      one tile exactly; one tile and a 1-pixel partial tile
  33x9              one pixel past a 32-wide and an 8-row CTA
  9x130             many tile rows in one partial tile column

At these sizes one texel is more than 0.1 % of an output, so the plain gate (99.9 % of texels) would fail between two legal
builds of the oracle.  Every pass is therefore held to its rounding floor: the kernels must agree with the oracle at least as
well as the "fma" and "uv" builds of the oracle do (parity.SideBySide, noise_floor).  Non-finite texels are never accepted."""
import pytest

from test_gpu_reblur import _dump  # the per-case JSON reports go where the other GPU parity tests write theirs

pytestmark = pytest.mark.gpu

SIZES = [(1, 1), (1, 64), (64, 1), (7, 5), (16, 16), (17, 17), (33, 9), (40, 3), (9, 130)]
EVERY_PASS = ("",)  # floor_passes: every shader name contains the empty string


def _settings(key):
    from raytracingdenoiser_b200 import nrd
    hd = nrd.HitDistanceReconstructionMode
    return {
        "default": None,
        "perf": lambda: nrd.ReblurSettings(enablePerformanceMode=True),
        "reblur_hitdist5x5": lambda: nrd.ReblurSettings(hitDistanceReconstructionMode=int(hd.AREA_5X5)),
        "reblur_antifirefly": lambda: nrd.ReblurSettings(enableAntiFirefly=True),
        "relax_antifirefly": lambda: nrd.RelaxSettings(enableAntiFirefly=True),
        "relax_hitdist3x3": lambda: nrd.RelaxSettings(hitDistanceReconstructionMode=int(hd.AREA_3X3)),
        "reblur_checkerboard": lambda: nrd.ReblurSettings(checkerboardMode=int(nrd.CheckerboardMode.BLACK)),
        "relax_checkerboard": lambda: nrd.RelaxSettings(checkerboardMode=int(nrd.CheckerboardMode.WHITE)),
    }[key]


# (denoiser, settings key, CommonSettings overrides)
CASES = [
    ("REBLUR_DIFFUSE_SPECULAR", "default", None),
    ("REBLUR_DIFFUSE_SPECULAR", "perf", None),
    ("REBLUR_DIFFUSE_SPECULAR", "reblur_hitdist5x5", None),
    ("REBLUR_DIFFUSE_SPECULAR", "reblur_antifirefly", None),
    ("REBLUR_DIFFUSE", "default", None),
    ("REBLUR_SPECULAR", "default", None),
    ("RELAX_DIFFUSE_SPECULAR", "default", None),
    ("RELAX_DIFFUSE_SPECULAR", "relax_antifirefly", None),
    ("RELAX_DIFFUSE_SPECULAR", "relax_hitdist3x3", None),
    ("RELAX_DIFFUSE", "default", None),
    ("RELAX_SPECULAR", "default", None),
    ("SIGMA_SHADOW", "default", None),
    ("SIGMA_SHADOW_TRANSLUCENCY", "default", None),
    ("REFERENCE", "default", None),
    ("REBLUR_DIFFUSE_SPECULAR", "default", {"splitScreen": 0.5}),
    ("RELAX_DIFFUSE_SPECULAR", "default", {"splitScreen": 0.5}),
    ("SIGMA_SHADOW", "default", {"splitScreen": 0.5}),
    ("REFERENCE", "default", {"splitScreen": 0.5}),
]
# checkerboarded inputs need an even width (scene.checkerboard_frame)
CHECKERBOARD = [("REBLUR_DIFFUSE_SPECULAR", "reblur_checkerboard", "BLACK"), ("RELAX_DIFFUSE_SPECULAR", "relax_checkerboard", "WHITE")]


def _params():
    out = []
    for w, h in SIZES:
        for den, key, common in CASES:
            cid = "%s-%s%s-%dx%d" % (den, key, "-split" if common else "", w, h)
            out.append(pytest.param(den, key, common, None, w, h, 0, id=cid))
        if w % 2 == 0:
            for den, key, mode in CHECKERBOARD:
                out.append(pytest.param(den, key, None, mode, w, h, 0, id="%s-%s-%dx%d" % (den, key, w, h)))
        for den in ("REBLUR_DIFFUSE_SPECULAR", "RELAX_DIFFUSE_SPECULAR"):  # steady state: HistoryFix skipped, antilag
            out.append(pytest.param(den, "default", None, None, w, h, 8, id="%s-warmup8-%dx%d" % (den, w, h)))
    return out


def _check(sbs, report, name):
    _dump(name, report)
    assert report, "no pass was compared"
    assert not sbs.failures(), sbs.describe_failures()


@pytest.mark.parametrize("denoiser_name,settings_key,common,checkerboard,width,height,warmup", _params())
def test_per_pass_parity_at_small_frame_sizes(denoiser_name, settings_key, common, checkerboard, width, height, warmup):
    """4 frames from frame 0 (the clears, young history), or 4 frames after 8 oracle-only frames (steady-state branches)."""
    import parity
    from raytracingdenoiser_b200 import nrd, scene
    settings_fn = _settings(settings_key)
    frame_fn = None
    if checkerboard:
        d, s = (0, 1) if checkerboard == "BLACK" else (1, 0)
        frame_fn = lambda fr, f: scene.checkerboard_frame(fr, f, d, s)  # noqa: E731
    sbs = parity.SideBySide(getattr(nrd.Denoiser, denoiser_name), width, height, settings=settings_fn() if settings_fn else None, common=common,
                            frame_fn=frame_fn, noise_floor=True, floor_passes=EVERY_PASS)
    report = sbs.run_per_pass(4, warmup=warmup)
    _check(sbs, report, "shapes_%s_%s%s%s_w%d_%dx%d.json" % (denoiser_name, settings_key, "_split" if common else "", "_" + checkerboard if checkerboard else "",
                                                             warmup, width, height))


def _edge_rects(f):
    """64x48 textures: full, the last texel, a rect touching the right and bottom edges, one smaller than a tile at the origin, full."""
    return [(0, 0, 64, 48), (63, 47, 1, 1), (40, 30, 24, 18), (0, 0, 17, 9), (0, 0, 64, 48)][f]


@pytest.mark.parametrize("denoiser_name", ["REBLUR_DIFFUSE_SPECULAR", "RELAX_DIFFUSE_SPECULAR", "SIGMA_SHADOW"])
def test_dynamic_resolution_rects_at_the_resource_edges(denoiser_name):
    """rectOrigin + rectSize at the right and bottom edges of the resource, a 1x1 rect, and a rect that shrinks and grows back."""
    import parity
    from raytracingdenoiser_b200 import nrd
    sbs = parity.SideBySide(getattr(nrd.Denoiser, denoiser_name), 64, 48, noise_floor=True, floor_passes=EVERY_PASS)
    report = sbs.run_per_pass(5, rect_fn=_edge_rects)
    assert {r["frame"] for r in report} == set(range(5))
    _check(sbs, report, "shapes_dynres_edges_%s.json" % denoiser_name)
