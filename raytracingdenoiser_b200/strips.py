"""Multi-GPU host logic: one process per GPU, the frame cut into horizontal strips of whole 16-row tiles.

Every rank runs the SAME pass list on its own strip (`nrd.CudaContext(strip=..., strip_height=...)`); rows of other strips
are read by the kernels straight from the owner's HBM over NVLink (CUDA IPC mapping of the owner's arena), and a device-side
flag barrier separates the passes (csrc/arena.cu).  There is no data-path collective: torch.distributed only carries the
64-byte IPC handles at start-up and the timing reductions of bench.py.
"""
import os

import torch

from . import harness, nrd

TILE = 16
# ghost rows each strip keeps of its neighbours (refreshed by bulk NVLink stores after every pass); taps beyond them are
# direct peer loads, so the value only trades halo traffic against the (slow) direct loads
DEFAULT_HALO_ROWS = int(os.environ.get("NRD_B200_HALO_ROWS", "96"))


def partition_rows(height, world_size):
    """Uniform strips of whole 16-row tiles: returns (strip_height, [(y0, y1)] per rank).  Every rank must own rows."""
    tiles = (height + TILE - 1) // TILE
    per_rank = (tiles + world_size - 1) // world_size
    strip_height = per_rank * TILE
    strips = [(r * strip_height, min((r + 1) * strip_height, height)) for r in range(world_size)]
    if any(y0 >= y1 for y0, y1 in strips):
        raise ValueError("a %d-row frame cannot be cut into %d strips of whole 16-row tiles" % (height, world_size))
    return strip_height, strips


def partition_rows_weighted(height, world_size, tile_row_cost, min_rows=TILE, max_rows=None):
    """Cost-balanced strips of whole 16-row tiles.  tile_row_cost[i] = estimated cost of tile row i (e.g. its number of
    non-sky tiles); returns (capacity, [(y0, y1)] per rank) with capacity = the tallest strip, to be passed as strip_height.
    Greedy prefix split: strip r ends at the first tile row where the running cost reaches (r + 1) / world_size of the total,
    subject to every strip holding at least `min_rows` rows and, if given, at most `max_rows` (the strip_height the contexts
    reserved: a re-cut for nrdCudaRepartition).  Raises ValueError when no cut satisfies both."""
    tiles = (height + TILE - 1) // TILE
    cost = [float(c) for c in tile_row_cost]
    assert len(cost) == tiles, (len(cost), tiles)
    min_tiles = max(1, (min_rows + TILE - 1) // TILE)
    if min_tiles * world_size > tiles:
        raise ValueError("a %d-row frame cannot be cut into %d strips of at least %d rows" % (height, world_size, min_rows))
    if max_rows is not None and (max_rows // TILE < min_tiles or max_rows // TILE * TILE * (world_size - 1) + max_rows < height):
        raise ValueError("a %d-row frame cannot be cut into %d strips of %d to %d rows" % (height, world_size, min_rows, max_rows))
    total = sum(cost) or 1.0
    bounds, acc, t = [0], 0.0, 0
    for r in range(world_size - 1):
        target = total * (r + 1) / world_size
        lo = bounds[-1] + min_tiles                          # this strip needs min_tiles rows ...
        hi = tiles - min_tiles * (world_size - 1 - r)        # ... and so does every strip after it
        if max_rows is not None:
            max_tiles = max_rows // TILE
            hi = min(hi, bounds[-1] + max_tiles)             # this strip fits max_rows ...
            rest = max_tiles * TILE * (world_size - 2 - r) + max_rows
            lo = max(lo, (height - rest + TILE - 1) // TILE)  # ... and so do the strips after it (the last may end mid-tile)
            if lo > hi:
                raise ValueError("a %d-row frame cannot be cut into %d strips of %d to %d rows" % (height, world_size, min_rows, max_rows))
        while t < lo or (t < hi and acc + 0.5 * cost[t] < target):
            acc += cost[t]
            t += 1
        bounds.append(t)
    bounds.append(tiles)
    strips = [(bounds[r] * TILE, min(bounds[r + 1] * TILE, height)) for r in range(world_size)]
    capacity = max((y1 - y0 + TILE - 1) // TILE * TILE for y0, y1 in strips)
    return capacity, strips


def tile_row_cost_from_viewz(viewz, denoising_range=500000.0):
    """Cost model of the partition: a 16x16 tile that is entirely beyond the denoising range is skipped by every pass
    (ClassifyTiles), all other tiles cost about the same.  viewz: (H, W) tensor of IN_VIEWZ; returns one cost per tile row."""
    h, w = viewz.shape
    th, tw = (h + TILE - 1) // TILE, (w + TILE - 1) // TILE
    pad = torch.full((th * TILE, tw * TILE), float("inf"), dtype=viewz.dtype, device=viewz.device)
    pad[:h, :w] = viewz.abs()
    live = (pad.view(th, TILE, tw, TILE).amin(dim=(1, 3)) <= denoising_range)
    return (live.float().sum(dim=1) + 0.02 * tw).tolist()   # a skipped tile still costs its early-out


def rebalance_tile_row_cost(tile_row_cost, strips, measured_ms):
    """Measured re-balancing: strips = [(y0, y1)] that were just run, measured_ms[r] = kernel time of rank r over them
    (nrdCudaGetTiming: kernels only, no barrier waits).  Returns the per-tile-row costs scaled strip by strip so that each
    strip's total is proportional to what it actually took; feeding them to partition_rows_weighted moves the boundaries
    towards equal time.  (The cost model only knows sky tiles; blur radii, young history, specular work per pixel are content.)"""
    cost = [float(c) for c in tile_row_cost]
    total_ms = float(sum(measured_ms)) or 1.0
    total_cost = sum(cost) or 1.0
    for (y0, y1), ms in zip(strips, measured_ms):
        t0, t1 = y0 // TILE, (y1 + TILE - 1) // TILE
        predicted = sum(cost[t0:t1])
        if predicted <= 0.0 or t1 <= t0:
            continue
        k = (ms / total_ms) / (predicted / total_cost)
        for t in range(t0, t1):
            cost[t] *= k
    return cost


def exchange_ipc_handles(local_handle, group=None):
    """all_gather of the per-rank 64-byte CUDA IPC handles (works on the gloo and the nccl backend)."""
    import torch.distributed as dist
    world = dist.get_world_size(group)
    on_gpu = dist.get_backend(group) == "nccl"
    dev = torch.device("cuda", torch.cuda.current_device()) if on_gpu else torch.device("cpu")
    mine = torch.tensor(list(local_handle), dtype=torch.uint8, device=dev)
    gathered = [torch.empty_like(mine) for _ in range(world)]
    dist.all_gather(gathered, mine, group=group)
    return [bytes(t.cpu().tolist()) for t in gathered]


class StripDenoiser(object):
    """The strip of one rank: instance + strip-mode CUDA context.  IN_*/OUT_* strips live in the context's arena.

    The strips can be re-cut between frames (repartition), keeping every history.  denoise() never does it by itself; a policy
    for dynamic resolution, where every pass produces only the rows above tiles(max(rectSize.y, rectSizePrev.y)):

        live = (max(rect_h, rect_h_prev) + 15) // 16                       # tile rows any pass of the frame produces
        if live != last_live:                                               # the same decision on every rank
            cost = [1.0 if t < live else 0.0 for t in range(tiles)]
            _, cut = partition_rows_weighted(height, world, cost, min_rows=halo, max_rows=part.strip_height)
            part.repartition(cut)                                           # before the frame's inputs are written
            last_live = live

    Reserve strip_height (the capacity) at creation for the most uneven cut wanted: the arena grows with it.  (REBLUR has a known
    gap on frames where the rect grows, with or without re-cuts: DESIGN.md section 6, tests/test_gpu_strips_rect_growth.py.)"""

    def __init__(self, denoiser, width, height, rank, world_size, device=0, identifier=0, settings=None, halo_rows=None, partition=None):
        """partition = (capacity, [(y0, y1)] per rank) from partition_rows_weighted; default: uniform strips."""
        self.denoiser, self.width, self.height, self.identifier = denoiser, width, height, identifier
        self.rank, self.world_size = rank, world_size
        self.device = torch.device("cuda", device)
        self.strip_height, strips = partition if partition is not None else partition_rows(height, world_size)
        self.strip_starts = [y0 for y0, _ in strips] + [height] if partition is not None else None
        self.y0, self.y1 = strips[rank]
        self.instance = nrd.Instance([(identifier, denoiser)])
        self.ctx = nrd.CudaContext(self.instance, width, height, device=device, strip=(self.y0, self.y1), strip_height=self.strip_height,
                                   halo_rows=DEFAULT_HALO_ROWS if halo_rows is None else halo_rows)
        if settings is not None:
            self.instance.set_denoiser_settings(identifier, settings)
        self.names = harness.DENOISER_RESOURCES[denoiser]

    def connect(self, group=None):
        """Multi-process: exchange the IPC handles over torch.distributed and map the peers' arenas."""
        handles = exchange_ipc_handles(self.ctx.ipc_handle(), group)
        self.ctx.connect_peers(self.rank, self.world_size, ipc_handles=handles, strip_starts=self.strip_starts)

    def connect_local(self, all_strips):
        """Single process (tests): every strip is a context of this process on a device that can address the others."""
        self.ctx.connect_peers(self.rank, self.world_size, arenas=[s.ctx.arena()[0] for s in all_strips], strip_starts=self.strip_starts)

    def repartition(self, strips, stream=None):
        """Collective between two frames (nrdCudaRepartition): every rank passes the same strips = [(y0, y1)] per rank, e.g. from
        partition_rows_weighted(..., max_rows=self.strip_height).  set_inputs / read_outputs copy the new rows afterwards."""
        if len(strips) != self.world_size or any(strips[r][1] != strips[r + 1][0] for r in range(self.world_size - 1)):
            raise ValueError("strips must be %d contiguous (y0, y1) pairs: %r" % (self.world_size, strips))
        starts = [y0 for y0, _ in strips] + [strips[-1][1]]
        self.ctx.repartition(starts, self._stream(stream))
        self.strip_starts = starts
        self.y0, self.y1 = strips[self.rank]

    def _stream(self, stream):
        return stream.cuda_stream if stream is not None else torch.cuda.current_stream(self.device).cuda_stream

    def set_inputs(self, frame, stream=None):
        """frame[name]: full-frame tensors (device or pinned host); only the rows of this strip are copied."""
        s = self._stream(stream)
        for name in self.names:
            if name.startswith("IN_"):
                t = frame[name][self.y0:self.y1]
                self.ctx.copy(getattr(nrd.ResourceType, name), 0, t.data_ptr(), t.stride(0) * t.element_size(), True, s)

    def set_input_strips(self, strips, stream=None):
        """strips[name]: tensors that hold exactly the rows of this strip."""
        s = self._stream(stream)
        for name, t in strips.items():
            self.ctx.copy(getattr(nrd.ResourceType, name), 0, t.data_ptr(), t.stride(0) * t.element_size(), True, s)

    def denoise(self, common_settings, stream=None):
        self.instance.set_common_settings(common_settings)
        return self.ctx.denoise([self.identifier], stream=self._stream(stream))

    def dispatches(self, common_settings):
        self.instance.set_common_settings(common_settings)
        r, raw, n = self.instance.get_compute_dispatches_raw([self.identifier])
        if r != nrd.Result.SUCCESS:
            raise nrd.NrdError("GetComputeDispatches", r)
        return raw, n

    def read_outputs(self, out=None, stream=None):
        """Copies the OUT_* strips into torch tensors (device by default, or the given pinned-host tensors)."""
        s = self._stream(stream)
        res = {}
        for name in self.names:
            if name.startswith("OUT_"):
                fmt, dtype, ch = harness.user_format(self.denoiser, name)
                rows = self.y1 - self.y0
                t = out[name] if out is not None else torch.empty((rows, self.width, ch) if ch > 1 else (rows, self.width), dtype=dtype, device=self.device)
                self.ctx.copy(getattr(nrd.ResourceType, name), 0, t.data_ptr(), t.stride(0) * t.element_size(), False, s)
                res[name] = t
        return res

    def synchronize(self, stream=None):
        self.ctx.synchronize(self._stream(stream))

    def destroy(self):
        self.ctx.destroy()
        self.instance.destroy()
