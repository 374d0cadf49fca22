// The device memory of a context and the multi-GPU strip exchange.
// Every texture a context owns is carved from one allocation, the arena: a header (barrier flags, error word, push ticket
// counter), then the textures, in the same layout on every rank.  Multi-GPU (strip mode, see include/nrd_b200.h): every texture
// is a strip of `stripHeight` rows plus ghost rows; arenas are exchanged with CUDA IPC and the kernels read foreign rows straight
// from the owner (device/common.cuh TexelPtr).  After every pass each rank pushes the rows it wrote next to its neighbours into
// their ghost rows, signals all its peers and waits for all of them: a pass may read what any rank wrote in the previous pass and
// may overwrite what any rank read in it.  The strip table can change between frames (Repartition): every texture keeps its place
// in the arena, only the rows it holds change.
#pragma once
#include "../../include/nrd_b200.h"
#include "device/surf.h"

#include <string>

namespace nrdb200
{
using namespace nrdb200_abi;

uint32_t BytesPerTexel(nrd::Format f);

struct Texture
{
    void* ptr = nullptr; // first row held locally: texel (0, firstRow - haloRows) in strip mode, texel (0, firstRow) otherwise
    size_t pitch = 0;
    nrd::Format format = nrd::Format::R8_UNORM;
    uint16_t width = 0, height = 0; // virtual size
    uint16_t firstRow = 0, rows = 0; // rows that hold data
    uint16_t allocRows = 0;          // rows of memory at ptr (in the arena in strip mode: uniform strip height + 2 x haloRows)
    uint16_t haloRows = 0;           // ghost rows above and below the strip, in this texture's own rows
    uint16_t downsample = 1;
    void* OwnPtr() const { return (uint8_t*)ptr + (size_t)haloRows * pitch; } // texel (0, firstRow)
    bool owned = false;              // in the arena; else an application texture (nrdCudaSetUserTexture)
};

struct StripState
{
    uint32_t rank = 0, world = 1;
    int peerSlot = -1;
    bool connected = false;
    void* peerArena[kMaxPeers] = {};
    bool peerOpened[kMaxPeers] = {};
    long long peerDelta[kMaxPeers] = {};
    uint32_t stripStart[kMaxPeers + 1] = {}; // first row of every rank's strip, [world] = frame height
    uint32_t epoch = 0;
    uint32_t halo = 0;               // ghost rows (full-resolution rows, multiple of 16, <= stripHeight)
    unsigned* hostError = nullptr;   // pinned + mapped: a strip barrier that timed out writes its epoch here (strip mode)
    bool MultiGpu() const { return world > 1; } // connected to other strips (nrdCudaConnectPeers)
};

// Calls that fail with a message return it in `error` (nrdCudaGetLastError).
struct Arena
{
    NrdCudaContextDesc desc{};
    uint8_t* base = nullptr;
    size_t bytes = 0;
    StripState strip;

    bool StripMode() const { return desc.stripHeight != 0; }
    // owned: a texture Allocate places in the arena; else an application texture at `ptr` with `pitch`
    Texture Describe(nrd::Format format, uint16_t downsample, bool owned, void* ptr = nullptr, size_t pitch = 0) const;
    Surf ToSurf(const Texture& t) const;
    nrd::Result Allocate(Texture* const* textures, size_t n); // places the owned ones in this order, allocates, zeroes
    void Release();
    nrd::Result ConnectPeers(const nrd::Instance& instance, uint32_t rank, uint32_t worldSize, const void* ipcHandles, void* const* arenas,
                             const uint16_t* stripStarts, std::string& error);
    // the rules of a strip table (worldSize + 1 first rows, the last = frame height) shared by ConnectPeers and Repartition
    nrd::Result CheckPartition(const uint32_t* starts, uint32_t worldSize, std::string& error) const;
    // Collective (nrdCudaRepartition): moves the rows of every owned texture in `textures` to their owners under the strip table
    // `stripStarts` (strip.world + 1 entries) and switches to it.  Enqueued on `stream` without a host synchronisation.
    nrd::Result Repartition(Texture* const* textures, size_t n, const uint16_t* stripStarts, cudaStream_t stream, std::string& error);
    // MultiGpu(): pushes the boundary rows of `textures`, just written by this rank, to the neighbours, then meets all ranks
    nrd::Result PushGhostsAndBarrier(const Texture* const* textures, uint32_t n, cudaStream_t stream, std::string& error);
    nrd::Result CheckBarriers(std::string& error) const; // fails if a barrier timed out
};

// Bit k set: output k of dispatches[i] needs fresh ghost rows, because a later pass reads it before anyone overwrites it, or
// because it survives the frame (not TRANSIENT_POOL) and may be read next frame.
uint32_t GhostPushMask(const nrd::DispatchDesc* dispatches, uint32_t n, uint32_t i);

cudaError_t LaunchClear(const PassLaunch& p);
} // namespace nrdb200
