"""Re-cutting connected strips between frames, the CPU side: partition_rows_weighted under a reserved strip height (max_rows), and
nrdCudaRepartition's argument check, which needs no device."""
import ctypes as C

import pytest


def _check_cut(height, world, cut, min_rows, max_rows):
    assert cut[0][0] == 0 and cut[-1][1] == height
    assert all(a[1] == b[0] for a, b in zip(cut, cut[1:]))
    assert all(y0 % 16 == 0 for y0, _ in cut)
    assert all(min_rows <= y1 - y0 <= max_rows for y0, y1 in cut[:-1])
    assert 0 < cut[-1][1] - cut[-1][0] <= max_rows


@pytest.mark.parametrize("height,world,halo,live_rows", [
    (2160, 2, 96, 1080),   # a 4K frame at a 1080p rect: the capacity lets the rect be split in two
    (2160, 4, 96, 1080),
    (2160, 3, 32, 720),
    (192, 4, 16, 48),      # the test frame of the GPU tests, a rect inside the first strip
    (1080, 2, 16, 1080),   # the full frame
    (141, 3, 16, 141),     # a last strip that ends mid-tile
])
def test_cut_of_the_live_rows_within_the_capacity(height, world, halo, live_rows):
    """Costs that are zero below the rows the passes produce: the live rows are shared within one tile of even, and every strip
    fits the capacity reserved for that cut."""
    from raytracingdenoiser_b200 import strips
    tiles = (height + 15) // 16
    live = (live_rows + 15) // 16
    cost = [1.0 if t < live else 0.0 for t in range(tiles)]
    # the capacity a context reserves for this cut: the live rows split evenly, the rest of the frame on the last rank
    even = (live + world - 1) // world * 16
    capacity = max(even + 16, -(-(height - even * (world - 1)) // 16) * 16)
    _, cut = strips.partition_rows_weighted(height, world, cost, min_rows=halo, max_rows=capacity)
    _check_cut(height, world, cut, max(halo, 16), capacity)
    share = [max(0, min(y1, live * 16) - y0) for y0, y1 in cut]
    assert max(share) - min(share) <= 16 + max(0, max(halo, 16) - live * 16 // world), (cut, share)


def test_a_tight_capacity_forces_the_cut():
    """All the cost in the first tile row: without max_rows one strip would take all but the minimum of the others; the capacity
    caps every strip and pushes the boundaries down."""
    from raytracingdenoiser_b200 import strips
    cost = [100.0] + [0.0] * 134
    _, free = strips.partition_rows_weighted(2160, 2, cost, min_rows=96)
    assert free == [(0, 96), (96, 2160)]
    _, capped = strips.partition_rows_weighted(2160, 2, cost, min_rows=96, max_rows=1200)
    assert capped == [(0, 960), (960, 2160)]
    _check_cut(2160, 2, capped, 96, 1200)
    _, exact = strips.partition_rows_weighted(2160, 3, [1.0] * 135, min_rows=96, max_rows=720)
    assert exact == [(0, 720), (720, 1440), (1440, 2160)]


@pytest.mark.parametrize("height,world,min_rows,max_rows", [
    (2160, 2, 96, 1072),   # two strips of at most 1072 rows cannot cover 2160
    (2160, 4, 96, 80),     # the capacity is below the minimum
    (192, 4, 64, 64),      # four strips of at least 64 rows need 256
])
def test_no_cut_fits(height, world, min_rows, max_rows):
    from raytracingdenoiser_b200 import strips
    with pytest.raises(ValueError):
        strips.partition_rows_weighted(height, world, [1.0] * ((height + 15) // 16), min_rows=min_rows, max_rows=max_rows)


def test_without_max_rows_the_cut_is_unchanged():
    """The cuts of the partition tests of test_multi_process.py, as they were before max_rows existed."""
    from raytracingdenoiser_b200 import strips
    sky = [1.0] * 18 + [60.0] * 117
    assert strips.partition_rows_weighted(2160, 2, sky, min_rows=96) == (1216, [(0, 1216), (1216, 2160)])
    assert strips.partition_rows_weighted(2160, 4, sky, min_rows=96) == (752, [(0, 752), (752, 1216), (1216, 1696), (1696, 2160)])
    assert strips.partition_rows_weighted(2160, 8, sky, min_rows=96) == (
        512, [(0, 512), (512, 752), (752, 992), (992, 1216), (1216, 1456), (1456, 1696), (1696, 1920), (1920, 2160)])
    flat = [1.0] * 135
    cap, part = strips.partition_rows_weighted(2160, 4, flat, min_rows=96)
    assert (cap, part) == (544, [(0, 544), (544, 1072), (1072, 1616), (1616, 2160)])
    ms = [2.0 * (y1 - y0) if r == 0 else 1.0 * (y1 - y0) for r, (y0, y1) in enumerate(part)]
    assert strips.partition_rows_weighted(2160, 4, strips.rebalance_tile_row_cost(flat, part, ms), min_rows=96) == (
        672, [(0, 336), (336, 816), (816, 1488), (1488, 2160)])
    assert strips.partition_rows_weighted(141, 3, [1.0] * 9) == (48, [(0, 48), (48, 96), (96, 141)])
    with pytest.raises(ValueError):
        strips.partition_rows_weighted(64, 8, [1.0] * 4)


def test_repartition_of_a_null_context_is_an_invalid_argument():
    from raytracingdenoiser_b200 import nrd
    starts = (C.c_uint16 * 3)(0, 96, 192)
    assert nrd._lib.nrdCudaRepartition(None, starts, None) == nrd.Result.INVALID_ARGUMENT
    assert nrd._lib.nrdCudaRepartition(None, None, None) == nrd.Result.INVALID_ARGUMENT
