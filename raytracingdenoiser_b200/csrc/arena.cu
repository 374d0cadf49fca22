// Arena placement, the strip exchange and their kernels (arena.h).
#include "arena.h"
#include "device/launch.h"
#include "constants.h"
#include "scheduler.h"

#include <cstring>
#include <mutex>

using namespace nrd;
using namespace nrdb200;

namespace
{
std::mutex g_slotMutex;
bool g_slotUsed[kMaxPeerSlots] = {};

constexpr int kSmCount = 132;                  // H100 SXM: caps the grids of the grid-stride clear / push kernels
// Arena header: barrier flags (kMaxPeers x u32, slot s = last epoch signalled by rank s), then the error word, and the ticket
// counter of the ghost push at word kPushCounterWord
constexpr size_t kArenaHeader = 256;
constexpr unsigned kErrorWord = kMaxPeers;
constexpr unsigned kPushCounterWord = 16;
constexpr long long kBarrierTimeoutNs = 2000000000ll; // 2 s of %globaltimer (independent of the SM clock): a missing peer turns into an error instead of a hung GPU

Result Fail(std::string& error, Result r, const std::string& msg)
{
    error = msg;
    return r;
}

size_t ArenaBytes(const Texture& t) { return (t.pitch * t.allocRows + 255) & ~(size_t)255; }

// Loads every kernel the instance's pipelines map to (see NRD_B200_LAUNCH): nothing may be loaded lazily once barriers spin.
void PreloadKernels(const Instance& instance, cudaError_t (*launchPass)(const PassLaunch&))
{
    alignas(16) static unsigned char dummy[1024] = {}; // a zeroed constant block big enough for every denoiser
    ((RelaxConstants*)dummy)->gDiffCheckerboard = ((RelaxConstants*)dummy)->gSpecCheckerboard = 2; // (checkerboard off; in preload mode every variant is loaded anyway)
    const nrdb200::Scheduler& scheduler = (const nrdb200::Scheduler&)instance;
    for (uint32_t i = 0; i < scheduler.GetDesc().pipelinesNum; i++)
    {
        PassLaunch p{};
        p.kind = scheduler.PipelineKind(i);
        p.constants = dummy;
        p.constantsSize = sizeof(dummy);
        p.gridW = p.gridH = 1;
        p.rowBegin = 0;
        p.rowEnd = 16;
        p.preloadOnly = true;
        (void)launchPass(p); // passes without a kernel are reported when they are dispatched
    }
}

struct BarrierArgs
{
    unsigned* flags; // local arena header
    long long delta[kMaxPeers];
    unsigned rank, world, epoch;
    long long timeout;        // nanoseconds of %globaltimer
    unsigned* hostError;      // pinned, device-mapped word of the context: a timed-out barrier reports here, the host sees it without a sync
};

struct PushItem
{
    const uint8_t* src;
    uint8_t* dst;
    unsigned long long bytes;
};
constexpr int kMaxPushItems = 32;
struct PushArgs
{
    PushItem items[kMaxPushItems];
};

// rows [firstRow, firstRow + rows) of t belong to the strip [y0, y1) (full-resolution rows)
void SetRows(Texture& t, uint32_t y0, uint32_t y1)
{
    int first = (int)y0 / t.downsample, last = ((int)y1 + t.downsample - 1) / t.downsample;
    if (last > (int)t.height) last = t.height;
    if (first > last) first = last;
    t.firstRow = (uint16_t)first;
    t.rows = (uint16_t)(last - first);
}

PeerTable MakePeerTable(const long long* peerDelta, const uint32_t* stripStart, uint32_t worldSize)
{
    PeerTable table{};
    for (uint32_t i = 0; i < (uint32_t)kMaxPeers; i++) table.delta[i] = peerDelta[i];
    for (uint32_t i = 0; i <= (uint32_t)kMaxPeers; i++) table.start[i] = i <= worldSize ? (int)stripStart[i] : 0x7fffffff;
    if (worldSize < (uint32_t)kMaxPeers) table.start[worldSize] = 0x7fffffff; // rows >= start[world] do not exist: never counted as an owner change
    return table;
}

// One owned texture of the repartition: where it lies in the texture region of every arena, and its rows under the new table.
struct MigrateItem
{
    unsigned long long offset; // from the start of the texture region (arena + kArenaHeader)
    unsigned pitch;            // a multiple of 256
    uint16_t height, allocRows, haloRows, downsample;
    uint16_t firstRow, rows;   // new
};
constexpr int kMaxMigrateItems = 128;
struct MigrateArgs
{
    const uint8_t* textures; // local texture region; a peer's is at + old.delta[peer]
    uint8_t* scratch;        // a copy of the texture region laid out like it, then the new table
    PeerTable* tableOut;
    PeerTable old, next;     // the strip tables before and after (the kernel must not read g_peerTable: it is switched later)
    unsigned n;
    MigrateItem items[kMaxMigrateItems];
};
} // namespace

namespace nrdb200
{
__global__ void ClearKernel(uint4* p, size_t n16)
{
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    size_t stride = (size_t)gridDim.x * blockDim.x;
    for (; i < n16; i += stride) p[i] = make_uint4(0, 0, 0, 0);
}

// Clear_Float / Clear_Uint: zero every texel of the (strip of the) texture.  Rows are 256-B multiples, so the whole
// allocation is cleared with 128-bit stores.
cudaError_t LaunchClear(const PassLaunch& p)
{
    const Surf& s = p.tex[0];
    size_t bytes = (size_t)s.pitch * (size_t)s.lrows; // ghost rows included: every rank clears them itself
    if (bytes == 0) return cudaSuccess;
    if ((s.pitch & 15) != 0 || ((uintptr_t)s.base & 15) != 0) return cudaMemsetAsync(s.base, 0, bytes, p.stream); // user textures with odd pitch
    size_t n16 = bytes / 16;
    int blocks = (int)((n16 + 255) / 256);
    if (blocks > kSmCount * 16) blocks = kSmCount * 16;
    if (blocks < 1) blocks = 1;
    ClearKernel<<<blocks, 256, 0, p.stream>>>((uint4*)s.base, n16);
    return cudaGetLastError();
}

__device__ __forceinline__ unsigned long long GlobalTimerNs()
{
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
__device__ __forceinline__ void StripBarrierBody(const BarrierArgs& a, unsigned t)
{
    if (t >= a.world) return;
    __threadfence_system();
    volatile unsigned* remote = (volatile unsigned*)((uint8_t*)a.flags + a.delta[t]) + a.rank;
    *remote = a.epoch;
    volatile unsigned* mine = a.flags + t;
    if (((volatile unsigned*)a.flags)[kErrorWord] != 0) return; // an earlier barrier of this context timed out: do not wait 2 s per pass again
    const unsigned long long start = GlobalTimerNs();
    while ((int)(*mine - a.epoch) < 0)
    {
        if ((long long)(GlobalTimerNs() - start) > a.timeout)
        {
            a.flags[kErrorWord] = a.epoch; // sticky error word (device side) ...
            if (a.hostError) *(volatile unsigned*)a.hostError = a.epoch; // ... and its host-visible twin: the next API call fails
            break;
        }
        __nanosleep(64);
    }
    __threadfence_system();
}

// All-to-all flag barrier over NVLink: lane t tells rank t "I finished epoch e" (a store into t's arena header) and then
// waits until rank t has told us the same.  Everything the previous kernel wrote is visible device-wide when this kernel
// starts (stream order); the system-scope fences order it against the flag for the remote readers.
__global__ void StripBarrierKernel(const __grid_constant__ BarrierArgs a) { StripBarrierBody(a, threadIdx.x); }

// Ghost refresh: after a pass wrote its strip of a texture, the first / last `halo` rows of the strip are stored into the
// ghost rows of the neighbour above / below (contiguous blocks of whole pitched rows, 16-byte NVLink stores).
// The block that finishes last also runs the inter-GPU barrier of this pass (one launch instead of two): every block fences
// its stores system-wide before it takes a ticket, the holder of the last ticket fences again and signals.
__global__ void __launch_bounds__(256) GhostPushKernel(const __grid_constant__ PushArgs a, const __grid_constant__ BarrierArgs b)
{
    const PushItem& it = a.items[blockIdx.y];
    const uint4* src = (const uint4*)it.src;
    uint4* dst = (uint4*)it.dst;
    const size_t n = it.bytes / 16;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) dst[i] = src[i];
    __shared__ unsigned last;
    __threadfence_system();
    __syncthreads();
    if (threadIdx.x == 0)
    {
        unsigned* counter = b.flags + kPushCounterWord;
        const unsigned ticket = atomicAdd(counter, 1u);
        last = ticket == gridDim.x * gridDim.y - 1 ? 1u : 0u;
        if (last) *counter = 0u; // ready for the next launch (stream order)
    }
    __syncthreads();
    if (last) StripBarrierBody(b, threadIdx.x);
}

// Repartition: texture blockIdx.y, local rows blockIdx.x, +gridDim.x, ... of its new layout.  A row of the new window (own rows and
// ghost rows inside the frame) is copied from the rank that owns it under the old table, where it is an own row; every other row
// (beyond the frame, or the unused tail of a strip shorter than the reserved height) is zeroed.  Rows are whole pitched rows,
// multiples of 256 B: 16-byte vectors whatever the format.  Downsampled textures count rows in their own units, as PeerRow does.
__global__ void __launch_bounds__(256) MigrateRowsKernel(const __grid_constant__ MigrateArgs a)
{
    if (blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0) *a.tableOut = a.next;
    const MigrateItem& it = a.items[blockIdx.y];
    const unsigned n16 = it.pitch / 16;
    const int window = (int)it.rows + 2 * (int)it.haloRows; // the rows kept current (Arena::ToSurf lrows)
    for (int k = blockIdx.x; k < (int)it.allocRows; k += gridDim.x)
    {
        const int y = (int)it.firstRow - (int)it.haloRows + k;
        const uint4* src = nullptr;
        if (k < window && y >= 0 && y < (int)it.height)
        {
            const int yFull = y * (int)it.downsample;
            int owner = 0;
#pragma unroll
            for (int j = 1; j < kMaxPeers; j++) owner += yFull >= a.old.start[j] ? 1 : 0;
            src = (const uint4*)(a.textures + a.old.delta[owner] + it.offset + (size_t)(y - a.old.start[owner] / (int)it.downsample + (int)it.haloRows) * it.pitch);
        }
        uint4* dst = (uint4*)(a.scratch + it.offset + (size_t)k * it.pitch);
        for (unsigned c = threadIdx.x; c < n16; c += blockDim.x) dst[c] = src ? src[c] : make_uint4(0, 0, 0, 0);
    }
}

uint32_t BytesPerTexel(Format f)
{
#define NRD_B200_BPT(name, bytes, isInt) bytes,
    static const uint32_t table[] = {NRD_B200_FORMATS(NRD_B200_BPT)};
#undef NRD_B200_BPT
    return (uint32_t)f < (uint32_t)Format::MAX_NUM ? table[(uint32_t)f] : 0;
}

Texture Arena::Describe(Format format, uint16_t downsample, bool owned, void* ptr, size_t pitch) const
{
    Texture t;
    t.format = format;
    t.downsample = downsample;
    t.width = uint16_t((desc.resourceWidth + downsample - 1) / downsample);
    t.height = uint16_t((desc.resourceHeight + downsample - 1) / downsample);
    SetRows(t, desc.stripY0, desc.stripY1);
    t.haloRows = uint16_t(strip.halo / downsample);
    t.allocRows = owned && StripMode() ? uint16_t(desc.stripHeight / downsample + 2 * t.haloRows) : t.rows;
    t.owned = owned;
    t.ptr = ptr; // owned: set by Allocate
    // 256-B aligned rows: 128-bit vector access and TMA-legal strides
    t.pitch = owned ? ((size_t)t.width * BytesPerTexel(format) + 255) & ~(size_t)255 : pitch;
    return t;
}

Surf Arena::ToSurf(const Texture& t) const
{
    // one GPU: the texture is the whole frame and all of it is local
    Surf s{};
    s.base = (uint8_t*)t.ptr;
    s.pitch = (int)t.pitch;
    s.w = t.width;
    s.h = t.height;
    s.y0 = t.firstRow;
    s.y1 = t.firstRow + t.rows;
    s.ly0 = t.firstRow;
    s.lrows = t.allocRows;
    if (strip.MultiGpu())
    {
        // connected strips: the kernels take the ghost-row / owner lookup for rows outside the strip
        s.stripRows = desc.stripHeight / t.downsample;
        s.rowShift = t.downsample == 16 ? 4u : 0u;
        s.halo = t.haloRows;
        s.ly0 = (int)t.firstRow - (int)t.haloRows;
        s.lrows = (unsigned)t.rows + 2u * t.haloRows; // the rows that are kept current: a strip shorter than the reserved height leaves the tail unused
        s.peerSlot = strip.peerSlot;
    }
    else if (StripMode())
        s.base += (size_t)t.haloRows * t.pitch, s.lrows = t.rows; // a strip context on its own holds the whole frame: skip its ghost rows
    return s;
}

Result Arena::Allocate(Texture* const* textures, size_t n)
{
    bytes = kArenaHeader;
    for (size_t i = 0; i < n; i++)
        if (textures[i]->owned) bytes += ArenaBytes(*textures[i]);
    if (cudaMalloc((void**)&base, bytes) != cudaSuccess) return base = nullptr, Result::FAILURE;
    size_t offset = kArenaHeader;
    for (size_t i = 0; i < n; i++)
        if (textures[i]->owned)
        {
            textures[i]->ptr = base + offset;
            offset += ArenaBytes(*textures[i]);
        }
    if (StripMode())
    {
        if (cudaHostAlloc((void**)&strip.hostError, sizeof(unsigned), cudaHostAllocMapped | cudaHostAllocPortable) != cudaSuccess)
            return strip.hostError = nullptr, Result::FAILURE;
        *strip.hostError = 0;
    }
    cudaMemset(base, 0, bytes);
    // the memset runs on the legacy default stream, the context is used on the caller's (non-blocking) streams and by peers:
    // nothing may touch the arena (barrier flags included) before it is zero
    cudaDeviceSynchronize();
    return Result::SUCCESS;
}

void Arena::Release()
{
    for (int i = 0; i < kMaxPeers; i++)
        if (strip.peerOpened[i]) cudaIpcCloseMemHandle(strip.peerArena[i]);
    if (strip.peerSlot >= 0)
    {
        std::lock_guard<std::mutex> lock(g_slotMutex);
        g_slotUsed[strip.peerSlot] = false;
    }
    if (base) cudaFree(base);
    if (strip.hostError) cudaFreeHost(strip.hostError);
}

Result Arena::ConnectPeers(const Instance& instance, uint32_t rank, uint32_t worldSize, const void* ipcHandles, void* const* arenas,
                           const uint16_t* stripStarts, std::string& error)
{
    if (worldSize == 0 || worldSize > (uint32_t)kMaxPeers || rank >= worldSize || (!ipcHandles == !arenas)) return Result::INVALID_ARGUMENT;
    if (!StripMode()) return Fail(error, Result::UNSUPPORTED, "not a strip-mode context");
    if (strip.connected) return Fail(error, Result::FAILURE, "peers already connected");
    StripState& s = strip;
    // strip starts: given explicitly (cost-aware partition) or uniform strips of stripHeight rows
    for (uint32_t i = 0; i <= worldSize; i++)
    {
        uint32_t y = stripStarts ? stripStarts[i] : i * (uint32_t)desc.stripHeight;
        if (!stripStarts && (i == worldSize || y > desc.resourceHeight)) y = desc.resourceHeight;
        s.stripStart[i] = y;
    }
    const Result pr = CheckPartition(s.stripStart, worldSize, error);
    if (pr != Result::SUCCESS) return pr;
    if (s.stripStart[rank] != desc.stripY0 || s.stripStart[rank + 1] != desc.stripY1) return Fail(error, Result::INVALID_ARGUMENT, "stripY0/stripY1 do not match the strip table");
    cudaSetDevice(desc.device);
    for (uint32_t i = 0; i < worldSize; i++)
    {
        if (i == rank) { s.peerArena[i] = base; continue; }
        if (arenas) s.peerArena[i] = arenas[i];
        else
        {
            cudaIpcMemHandle_t h;
            memcpy(&h, (const uint8_t*)ipcHandles + (size_t)i * sizeof(h), sizeof(h));
            cudaError_t e = cudaIpcOpenMemHandle(&s.peerArena[i], h, cudaIpcMemLazyEnablePeerAccess);
            if (e != cudaSuccess) return Fail(error, Result::FAILURE, std::string("cudaIpcOpenMemHandle: ") + cudaGetErrorString(e));
            s.peerOpened[i] = true;
        }
    }
    for (uint32_t i = 0; i < (uint32_t)kMaxPeers; i++) s.peerDelta[i] = i < worldSize ? (long long)((uint8_t*)s.peerArena[i] - base) : 0;
    {
        std::lock_guard<std::mutex> lock(g_slotMutex);
        for (int k = 0; k < kMaxPeerSlots && s.peerSlot < 0; k++)
            if (!g_slotUsed[k]) { g_slotUsed[k] = true; s.peerSlot = k; }
    }
    if (s.peerSlot < 0) return Fail(error, Result::FAILURE, "too many strip-mode contexts in one process");
    const PeerTable table = MakePeerTable(s.peerDelta, s.stripStart, worldSize);
    cudaError_t e = SetPeerTables(s.peerSlot, &table);
    if (e != cudaSuccess) return Fail(error, Result::FAILURE, std::string("peer table: ") + cudaGetErrorString(e));
    s.rank = rank;
    s.world = worldSize;
    s.connected = true;
    PreloadKernels(instance, worldSize > 1 ? nrdb200::LaunchPass : nrdb200_single::LaunchPass);
    // The arena's own kernels are preloaded too: the stand-alone barrier is first needed by a pass that pushes nothing, i.e.
    // possibly while this rank's previous (fused) barrier still spins for a peer whose launches the host has not issued yet --
    // a lazy load at that point would wait for the spinning kernel.
    cudaFuncAttributes fa;
    (void)cudaFuncGetAttributes(&fa, ClearKernel);
    (void)cudaFuncGetAttributes(&fa, StripBarrierKernel);
    (void)cudaFuncGetAttributes(&fa, GhostPushKernel);
    (void)cudaFuncGetAttributes(&fa, MigrateRowsKernel);
    return Result::SUCCESS;
}

Result Arena::CheckPartition(const uint32_t* starts, uint32_t worldSize, std::string& error) const
{
    if (starts[0] != 0 || starts[worldSize] != desc.resourceHeight) return Fail(error, Result::INVALID_ARGUMENT, "the strips do not cover the frame");
    for (uint32_t i = 0; i < worldSize; i++)
    {
        const uint32_t rows = starts[i + 1] - starts[i];
        if (starts[i + 1] <= starts[i] || starts[i] % 16 != 0 || rows > desc.stripHeight)
            return Fail(error, Result::INVALID_ARGUMENT, "every strip must start on a multiple of 16, own rows and fit stripHeight");
        if (rows < strip.halo && i + 1 < worldSize) return Fail(error, Result::INVALID_ARGUMENT, "haloRows exceeds the height of a strip (ghost rows are refreshed by the direct neighbours only)");
    }
    return Result::SUCCESS;
}

// Order on `stream`, the same on every rank:
//   barrier A   the previous frame's writes of every rank are complete and visible
//   MigrateRowsKernel   every row the new partition holds here (own and ghost rows), read from its owner under the OLD table,
//               into a scratch copy of the texture region; rows outside the frame and the unused tail of a strip read 0
//   barrier B   no rank still reads the old layout
//   copy back, scratch -> arena; the new table into every kernel translation unit (stream-ordered: the kernels queued before
//               still read the old one); the scratch is freed
//   barrier C   no peer pushes ghost rows (the next frame start) into rows the copy-back still writes
// Every allocation and copy is stream-ordered: in one process, ranks are contexts of one GPU, and a host call that waits for the
// device would wait for a barrier spinning for a rank the host has not reached yet.
Result Arena::Repartition(Texture* const* textures, size_t n, const uint16_t* stripStarts, cudaStream_t stream, std::string& error)
{
    if (!StripMode() || !strip.connected) return Fail(error, Result::UNSUPPORTED, "not a connected strip-mode context");
    if (strip.hostError && *(volatile unsigned*)strip.hostError)
        return Fail(error, Result::FAILURE, "a strip barrier of this context timed out waiting for a peer (epoch " + std::to_string(*(volatile unsigned*)strip.hostError) + ")");
    StripState& s = strip;
    uint32_t starts[kMaxPeers + 1] = {};
    for (uint32_t i = 0; i <= s.world; i++) starts[i] = stripStarts[i];
    const Result pr = CheckPartition(starts, s.world, error);
    if (pr != Result::SUCCESS || !s.MultiGpu()) return pr; // a world of one: the identity table is the only valid one
    MigrateArgs a{};
    a.textures = base + kArenaHeader;
    a.old = MakePeerTable(s.peerDelta, s.stripStart, s.world);
    a.next = MakePeerTable(s.peerDelta, starts, s.world);
    uint32_t maxRows = 0;
    for (size_t i = 0; i < n; i++)
    {
        const Texture& t = *textures[i];
        if (!t.owned) continue;
        if (a.n == (uint32_t)kMaxMigrateItems) return Fail(error, Result::FAILURE, "repartition: more textures than one launch carries (" + std::to_string(kMaxMigrateItems) + ")");
        Texture moved = t;
        SetRows(moved, starts[s.rank], starts[s.rank + 1]);
        a.items[a.n++] = {(unsigned long long)((uint8_t*)t.ptr - a.textures), (unsigned)t.pitch, t.height, t.allocRows, t.haloRows, t.downsample, moved.firstRow, moved.rows};
        if (t.allocRows > maxRows) maxRows = t.allocRows;
    }
    const size_t region = bytes - kArenaHeader; // every owned texture, in arena order (256-B multiples)
    // (the pool of the stream's device: the caller's current device, as for every other call of the executor)
    cudaError_t e = cudaMallocAsync((void**)&a.scratch, region + sizeof(PeerTable), stream);
    if (e != cudaSuccess) return Fail(error, Result::FAILURE, std::string("repartition scratch: ") + cudaGetErrorString(e));
    a.tableOut = (PeerTable*)(a.scratch + region);
    Result r = PushGhostsAndBarrier(nullptr, 0, stream, error); // A
    if (r == Result::SUCCESS)
    {
        MigrateRowsKernel<<<dim3(maxRows < 256u ? maxRows : 256u, a.n), 256, 0, stream>>>(a);
        e = cudaGetLastError();
        if (e != cudaSuccess) r = Fail(error, Result::FAILURE, std::string("repartition: ") + cudaGetErrorString(e));
    }
    if (r == Result::SUCCESS) r = PushGhostsAndBarrier(nullptr, 0, stream, error); // B
    if (r == Result::SUCCESS)
    {
        e = cudaMemcpyAsync(base + kArenaHeader, a.scratch, region, cudaMemcpyDeviceToDevice, stream);
        if (e == cudaSuccess) e = SetPeerTables(s.peerSlot, a.tableOut, &stream);
        if (e != cudaSuccess) r = Fail(error, Result::FAILURE, std::string("repartition: ") + cudaGetErrorString(e));
    }
    e = cudaFreeAsync(a.scratch, stream);
    if (r != Result::SUCCESS) return r;
    if (e != cudaSuccess) return Fail(error, Result::FAILURE, std::string("repartition: ") + cudaGetErrorString(e));
    // the host side of the new table: what every later launch, push and nrdCudaGetTexture sees
    for (uint32_t i = 0; i <= s.world; i++) s.stripStart[i] = starts[i];
    desc.stripY0 = (uint16_t)starts[s.rank];
    desc.stripY1 = (uint16_t)starts[s.rank + 1];
    for (size_t i = 0; i < n; i++)
        if (textures[i]->owned) SetRows(*textures[i], desc.stripY0, desc.stripY1);
    return PushGhostsAndBarrier(nullptr, 0, stream, error); // C
}

Result Arena::PushGhostsAndBarrier(const Texture* const* textures, uint32_t n, cudaStream_t stream, std::string& error)
{
    if (!strip.MultiGpu()) return Result::SUCCESS;
    const StripState& s = strip;
    PushArgs a{};
    uint32_t items = 0;
    unsigned long long maxBytes = 0;
    const uint32_t itemsPerTexture = (s.rank > 0 ? 1u : 0u) + (s.rank + 1 < s.world ? 1u : 0u);
    for (uint32_t i = 0; i < n; i++)
    {
        const Texture& t = *textures[i];
        if (!t.owned || !t.rows || !t.haloRows) continue;
        if (items + itemsPerTexture > (uint32_t)kMaxPushItems)
            return Fail(error, Result::FAILURE, "ghost push: more textures to push than one launch carries (" + std::to_string(kMaxPushItems) + " strip edges)");
        const uint32_t H = t.haloRows, cnt = t.rows < H ? t.rows : H; // ConnectPeers guarantees rows >= H except for the last strip
        const unsigned long long bytesPerSide = (unsigned long long)cnt * t.pitch;
        uint8_t* p = (uint8_t*)t.ptr;
        // my first rows are the bottom ghost rows of the strip above: they follow its own rows, i.e. local rows [H + rowsAbove, ...) there
        if (s.rank > 0)
            a.items[items++] = {p + (size_t)H * t.pitch, p + s.peerDelta[s.rank - 1] + (size_t)(H + (s.stripStart[s.rank] - s.stripStart[s.rank - 1]) / t.downsample) * t.pitch, bytesPerSide};
        // my last rows are the top ghost rows of the strip below: local rows [H - cnt, H) over there
        if (s.rank + 1 < s.world) a.items[items++] = {p + (size_t)(H + t.rows - cnt) * t.pitch, p + s.peerDelta[s.rank + 1] + (size_t)(H - cnt) * t.pitch, bytesPerSide};
        if (bytesPerSide > maxBytes) maxBytes = bytesPerSide;
    }
    BarrierArgs b{(unsigned*)base, {}, s.rank, s.world, ++strip.epoch, kBarrierTimeoutNs, s.hostError};
    for (uint32_t i = 0; i < s.world; i++) b.delta[i] = s.peerDelta[i];
    unsigned blocksX = (unsigned)((maxBytes / 16 + 256 * 8 - 1) / (256 * 8)); // ~8 x 16 B per thread
    if (blocksX < 1) blocksX = 1;
    if (blocksX > kSmCount * 4) blocksX = kSmCount * 4;
    if (items) GhostPushKernel<<<dim3(blocksX, items), 256, 0, stream>>>(a, b); // one push launch carries the barrier
    else StripBarrierKernel<<<1, 32, 0, stream>>>(b);
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? Result::SUCCESS : Fail(error, Result::FAILURE, std::string(items ? "ghost push: " : "strip barrier: ") + cudaGetErrorString(e));
}

Result Arena::CheckBarriers(std::string& error) const
{
    if (!strip.MultiGpu()) return Result::SUCCESS;
    unsigned err = 0;
    const cudaError_t e = cudaMemcpy(&err, base + sizeof(unsigned) * kErrorWord, sizeof(err), cudaMemcpyDeviceToHost);
    if (e != cudaSuccess) return Fail(error, Result::FAILURE, cudaGetErrorString(e));
    if (err) return Fail(error, Result::FAILURE, "strip barrier timed out waiting for a peer (epoch " + std::to_string(err) + ")");
    return Result::SUCCESS;
}

uint32_t GhostPushMask(const DispatchDesc* dispatches, uint32_t n, uint32_t i)
{
    uint32_t mask = 0;
    const DispatchDesc& d = dispatches[i];
    for (uint32_t k = 0; k < d.resourcesNum && k < 32; k++)
    {
        const ResourceDesc& out = d.resources[k];
        if (out.descriptorType != DescriptorType::STORAGE_TEXTURE) continue;
        // the first later dispatch that binds the texture decides; a pass may bind a texture both ways (never in the supported
        // chains): reading wins
        bool bound = false, read = false;
        for (uint32_t j = i + 1; j < n && !bound; j++)
            for (uint32_t m = 0; m < dispatches[j].resourcesNum; m++)
            {
                const ResourceDesc& use = dispatches[j].resources[m];
                if (use.type != out.type || use.indexInPool != out.indexInPool) continue;
                bound = true;
                read |= use.descriptorType == DescriptorType::TEXTURE;
            }
        // nothing later in the frame binds it: history, or an output a denoiser re-reads next frame (SIGMA)
        if (bound ? read : out.type != ResourceType::TRANSIENT_POOL) mask |= 1u << k;
    }
    return mask;
}
} // namespace nrdb200
