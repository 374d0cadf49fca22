"""A known gap of strip mode under dynamic resolution, with no re-cut anywhere: REBLUR temporal accumulation on the frame where the
rect grows back after frames at a smaller rect.  The history footprint of a pixel sits at its position scaled by
rectSizePrev / rectSize, so right below a strip boundary it lies far above the pixel; beyond the ghost rows the strip build's
output then differs from one context in a few texels of the first rows of the lower strip.  With a halo that holds the whole
other strip every footprint is local and the frames match; with a 16-row halo they do not (strict xfail: the test starts to
fail, and must be turned into a plain test, once the gap is fixed).  Same harness as test_gpu_strips_repartition.py."""
import pytest

pytestmark = pytest.mark.gpu

RECTS = [(0, 0, 320, 192), (0, 0, 320, 192), (0, 0, 200, 40), (0, 0, 200, 40), (0, 0, 250, 100), (0, 0, 320, 192)]


def _run(halo):
    import os
    import test_gpu_strips_repartition as T
    os.environ["NRD_B200_FORCE_STRIP_KERNELS"] = "1"
    rig = None
    try:
        rig = T._Rig("REBLUR_DIFFUSE_SPECULAR", 2, halo, first_cut=[(0, 96), (96, 192)], capacity=96)
        for f, rect in enumerate(RECTS):
            rig.frame(f, rect, RECTS[f - 1] if f else rect)
    finally:
        if rig is not None:
            rig.destroy()
        del os.environ["NRD_B200_FORCE_STRIP_KERNELS"]


def test_growing_rect_with_a_halo_that_holds_the_other_strip():
    _run(96)


@pytest.mark.xfail(strict=True, reason="REBLUR temporal accumulation, growing rect: history footprints beyond the ghost rows differ "
                                      "from one context (DESIGN.md section 6)")
def test_growing_rect_with_a_16_row_halo():
    _run(16)
