// CUDA executor: owns the pool textures in HBM and turns DispatchDesc[] into sm_90a kernel launches.
// Takes the role of the reference's optional NRI integration layer (Integration/NRDIntegration.hpp: pool creation
// :292-363, Denoise :516-623, Dispatch :625-803).  Stream order replaces the SRV/UAV barriers (:667-704); constants
// travel as __grid_constant__ kernel parameters instead of a constant-buffer ring (:721-749).
//
// Multi-GPU (strip mode, see include/nrd_b200.h): every texture of a context is a strip of `stripHeight` rows carved from
// one arena; arenas are exchanged with CUDA IPC and the kernels read foreign rows straight from the owner (common.cuh
// TexelPtr).  Between two passes every rank signals all its peers and waits for all of them (StripBarrierKernel): a pass
// may read what any rank wrote in the previous pass and may overwrite what any rank read in it.
#include "../../include/nrd_b200.h"
#include "device/launch.h"
#include "constants.h"
#include "scheduler.h"

#include <atomic>
#include <cstdio>
#include <cstring>
#include <mutex>
#include <string>
#include <vector>

using namespace nrd;
using namespace nrdb200;

namespace nrdb200
{
cudaError_t LaunchClear(const PassLaunch& p);
}

namespace
{
std::atomic<uint64_t> g_launchCount{0};
std::mutex g_slotMutex;
bool g_slotUsed[kMaxPeerSlots] = {};

constexpr int kSmCount = 132;                  // H100 SXM: caps the grids of the grid-stride copy / clear kernels
constexpr size_t kArenaHeader = 256;          // barrier flags: kMaxPeers x u32 (slot s = last epoch signalled by rank s), then the error word
constexpr unsigned kPushCounterWord = 16;      // u32 index in the header: ticket counter of the fused ghost push + barrier kernel
constexpr long long kBarrierTimeoutNs = 2000000000ll; // 2 s of %globaltimer (independent of the SM clock): a missing peer turns into an error instead of a hung GPU

uint32_t BytesPerTexel(Format f)
{
#define NRD_B200_BPT(name, bytes, isInt) bytes,
    static const uint32_t table[] = {NRD_B200_FORMATS(NRD_B200_BPT)};
#undef NRD_B200_BPT
    return (uint32_t)f < (uint32_t)Format::MAX_NUM ? table[(uint32_t)f] : 0;
}

struct Texture
{
    void* ptr = nullptr; // first row held locally: texel (0, firstRow - haloRows) in strip mode, texel (0, firstRow) otherwise
    size_t pitch = 0;
    Format format = Format::R8_UNORM;
    uint16_t width = 0, height = 0; // virtual size
    uint16_t firstRow = 0, rows = 0; // rows that hold data
    uint16_t allocRows = 0;          // rows reserved in the arena (strip mode: uniform strip height + 2 x haloRows)
    uint16_t haloRows = 0;           // ghost rows above and below the strip, in this texture's own rows
    uint16_t downsample = 1;
    void* OwnPtr() const { return (uint8_t*)ptr + (size_t)haloRows * pitch; } // texel (0, firstRow)
    bool owned = false;
};

// user textures the supported denoisers consume, with the one format the kernels are written for
// (OUT_SHADOW_TRANSLUCENCY: R8 for SIGMA_SHADOW, RGBA8 for SIGMA_SHADOW_TRANSLUCENCY -- `translucent` picks)
bool ExpectedUserFormat(ResourceType type, Format& expected, bool translucent = false)
{
    switch (type)
    {
        case ResourceType::IN_TRANSLUCENCY: expected = Format::RGBA8_UNORM; return true;
        case ResourceType::IN_MV: expected = Format::RGBA16_SFLOAT; return true;
        case ResourceType::IN_NORMAL_ROUGHNESS: expected = Format::R10_G10_B10_A2_UNORM; return true;
        case ResourceType::IN_VIEWZ: expected = Format::R32_SFLOAT; return true;
        case ResourceType::IN_DIFF_RADIANCE_HITDIST:
        case ResourceType::IN_SPEC_RADIANCE_HITDIST:
        case ResourceType::OUT_DIFF_RADIANCE_HITDIST:
        case ResourceType::OUT_SPEC_RADIANCE_HITDIST: expected = Format::RGBA16_SFLOAT; return true;
        case ResourceType::IN_PENUMBRA: expected = Format::R16_SFLOAT; return true;
        case ResourceType::IN_SIGNAL:
        case ResourceType::OUT_SIGNAL: expected = Format::RGBA16_SFLOAT; return true; // REFERENCE denoiser
        // optional inputs (CommonSettings::isHistoryConfidenceAvailable / isDisocclusionThresholdMixAvailable)
        case ResourceType::IN_DIFF_CONFIDENCE:
        case ResourceType::IN_SPEC_CONFIDENCE:
        case ResourceType::IN_DISOCCLUSION_THRESHOLD_MIX: expected = Format::R8_UNORM; return true;
        case ResourceType::IN_BASECOLOR_METALNESS: expected = Format::RGBA8_UNORM; return true; // CommonSettings::isBaseColorMetalnessAvailable
        case ResourceType::OUT_SHADOW_TRANSLUCENCY: expected = translucent ? Format::RGBA8_UNORM : Format::R8_UNORM; return true;
        default: return false;
    }
}
} // namespace

// ---- user textures in a format above the minimum (Include/NRDDescs.h:43-137 lists MINIMUM formats) -----------------------------------
// The kernels are written for one format per user texture (ExpectedUserFormat).  A texture bound in a wider format of the same kind
// (e.g. RGBA32_SFLOAT radiance, R16_SFLOAT viewZ, RG16_SFLOAT motion) gets a shadow copy in the kernels' format: inputs are converted
// into it before the passes that read them, outputs out of it after the passes that wrote them (one streaming kernel per texture).
struct FormatInfo
{
    int channels;
    int kind; // 0 = UNORM8, 1 = SFLOAT16, 2 = SFLOAT32
};
bool ConvertibleFormat(Format f, FormatInfo& info)
{
    switch (f)
    {
        case Format::R8_UNORM: info = {1, 0}; return true;
        case Format::RGBA8_UNORM: info = {4, 0}; return true;
        case Format::R16_SFLOAT: info = {1, 1}; return true;
        case Format::RG16_SFLOAT: info = {2, 1}; return true;
        case Format::RGBA16_SFLOAT: info = {4, 1}; return true;
        case Format::R32_SFLOAT: info = {1, 2}; return true;
        case Format::RG32_SFLOAT: info = {2, 2}; return true;
        case Format::RGBA32_SFLOAT: info = {4, 2}; return true;
        default: return false;
    }
}
struct ConvertArgs
{
    const uint8_t* src;
    uint8_t* dst;
    size_t srcPitch, dstPitch;
    int width, height;
    int srcChannels, srcKind, dstChannels, dstKind;
};
__device__ __forceinline__ float LoadChannel(const uint8_t* texel, int kind, int ch)
{
    if (kind == 0) return (float)texel[ch] / 255.0f;
    if (kind == 1) return __half2float(__ushort_as_half(((const unsigned short*)texel)[ch]));
    return ((const float*)texel)[ch];
}
__device__ __forceinline__ void StoreChannel(uint8_t* texel, int kind, int ch, float v)
{
    if (kind == 0) texel[ch] = (unsigned char)__fadd_rn(__fmul_rn(__saturatef(v), 255.0f), 0.5f); // D3D float -> UNORM
    else if (kind == 1) ((unsigned short*)texel)[ch] = __half_as_ushort(__float2half_rn(v));
    else ((float*)texel)[ch] = v;
}
// channels the source does not have read 0 (a two-channel motion vector has no z / w), extra source channels are dropped
__global__ void __launch_bounds__(256) ConvertFormatKernel(const __grid_constant__ ConvertArgs a)
{
    const int x = blockIdx.x * 32 + threadIdx.x, y = blockIdx.y * 8 + threadIdx.y;
    if (x >= a.width || y >= a.height) return;
    const int srcBytes = a.srcChannels * (a.srcKind == 0 ? 1 : (a.srcKind == 1 ? 2 : 4)), dstBytes = a.dstChannels * (a.dstKind == 0 ? 1 : (a.dstKind == 1 ? 2 : 4));
    const uint8_t* s = a.src + (size_t)y * a.srcPitch + (size_t)x * srcBytes;
    uint8_t* d = a.dst + (size_t)y * a.dstPitch + (size_t)x * dstBytes;
    for (int ch = 0; ch < a.dstChannels; ch++) StoreChannel(d, a.dstKind, ch, ch < a.srcChannels ? LoadChannel(s, a.srcKind, ch) : 0.0f);
}
struct ForeignTexture
{
    void* ptr = nullptr;     // the application's texture
    size_t pitch = 0;
    Format format = Format::R8_UNORM;
    void* shadow = nullptr;  // cudaMalloc'ed copy in the kernels' format (NrdCudaContext::user[] points at it)
};

struct NrdCudaContext
{
    Instance* instance = nullptr;
    NrdCudaContextDesc desc{};
    uint8_t* arena = nullptr;
    size_t arenaBytes = 0;
    std::vector<Texture> permanent, transient;
    Texture user[(size_t)ResourceType::MAX_NUM];
    ForeignTexture foreign[(size_t)ResourceType::MAX_NUM]; // user textures bound in a wider format than the kernels' (see ConvertFormatKernel)
    // decoded-guide surface of the REBLUR spatial passes (surf.h PassLaunch::guide): written by ClassifyTiles, the first pass
    // of every REBLUR frame, read by PrePass / Blur / PostBlur of the same frame
    Texture guide;
    bool guideValid = false;
    // roughness table of the REBLUR spatial passes (surf.h PassLaunch::roughnessLut), rebuilt when hitDistanceParameters change
    float* roughnessLut = nullptr;     // device, 1024 x float4 (allocated with the context: no cudaMalloc -- an implicit device
    float* roughnessLutStaging = nullptr; // synchronisation -- may happen while a strip barrier spins); pinned staging copy
    cudaEvent_t lutUploaded = nullptr;
    unsigned* hostError = nullptr;        // pinned + mapped: a strip barrier that timed out writes its epoch here (strip mode)
    bool timing = false;                  // nrdCudaSetTiming: three events per dispatch (before the kernel, after it, after push + barrier)
    cudaEvent_t timingEvents[3 * 64] = {};
    uint32_t timingCount = 0;
    float lutKey[2] = {0.0f, 0.0f};
    bool lutValid = false;
    // strip mode
    uint32_t rank = 0, world = 1;
    int peerSlot = -1;
    bool connected = false;
    void* peerArena[kMaxPeers] = {};
    bool peerOpened[kMaxPeers] = {};
    long long peerDelta[kMaxPeers] = {};
    uint32_t stripStart[kMaxPeers + 1] = {}; // first row of every rank's strip, [world] = frame height
    uint32_t epoch = 0;
    uint32_t halo = 0; // ghost rows (full-resolution rows, multiple of 16, <= stripHeight)
    std::string lastError;
};

namespace
{
Result Fail(NrdCudaContext* ctx, Result r, const std::string& msg)
{
    if (ctx) ctx->lastError = msg;
    return r;
}

bool StripMode(const NrdCudaContext* ctx) { return ctx->desc.stripHeight != 0; }

// rows [first, first + rows) of a texture with `downsample` that belong to the context
void OwnedRows(const NrdCudaContextDesc& d, uint16_t downsample, uint16_t virtualHeight, uint16_t& first, uint16_t& rows)
{
    int f = d.stripY0 / downsample, l = (d.stripY1 + downsample - 1) / downsample;
    if (l > (int)virtualHeight) l = virtualHeight;
    if (f > l) f = l;
    first = (uint16_t)f;
    rows = (uint16_t)(l - f);
}

void DescribeTexture(const NrdCudaContext* ctx, Format format, uint16_t downsample, Texture& t)
{
    t.format = format;
    t.downsample = downsample;
    t.width = uint16_t((ctx->desc.resourceWidth + downsample - 1) / downsample);
    t.height = uint16_t((ctx->desc.resourceHeight + downsample - 1) / downsample);
    OwnedRows(ctx->desc, downsample, t.height, t.firstRow, t.rows);
    t.haloRows = uint16_t(ctx->halo / downsample);
    t.allocRows = StripMode(ctx) ? uint16_t(ctx->desc.stripHeight / downsample + 2 * t.haloRows) : t.rows;
    size_t rowBytes = (size_t)t.width * BytesPerTexel(format);
    t.pitch = (rowBytes + 255) & ~(size_t)255; // 256-B aligned rows: 128-bit vector access and TMA-legal strides
    t.owned = true;
}

const Texture* Resolve(NrdCudaContext* ctx, ResourceType type, uint32_t index)
{
    if (type == ResourceType::PERMANENT_POOL) return index < ctx->permanent.size() ? &ctx->permanent[index] : nullptr;
    if (type == ResourceType::TRANSIENT_POOL) return index < ctx->transient.size() ? &ctx->transient[index] : nullptr;
    if ((uint32_t)type < (uint32_t)ResourceType::MAX_NUM && ctx->user[(uint32_t)type].ptr) return &ctx->user[(uint32_t)type];
    return nullptr;
}

Surf ToSurf(const NrdCudaContext* ctx, const Texture& t)
{
    Surf s{};
    s.base = (uint8_t*)t.ptr;
    s.pitch = (int)t.pitch;
    s.w = t.width;
    s.h = t.height;
    s.y0 = t.firstRow;
    s.y1 = t.firstRow + t.rows;
    s.ly0 = t.firstRow;
    s.lrows = t.owned ? t.allocRows : t.rows;
    if (StripMode(ctx) && ctx->world > 1)
    {
        s.stripRows = ctx->desc.stripHeight / t.downsample;
        s.rowShift = t.downsample == 16 ? 4u : 0u;
        s.halo = t.haloRows;
        s.ly0 = (int)t.firstRow - (int)t.haloRows;
        s.lrows = (unsigned)t.rows + 2u * t.haloRows; // the rows that are kept current: a strip shorter than the reserved height leaves the tail unused
        s.peerSlot = ctx->peerSlot;
    }
    else if (StripMode(ctx))
        s.base += (size_t)t.haloRows * t.pitch, s.lrows = t.rows; // a strip-mode context that holds the whole frame
    return s;
}

// WithRectOrigin (Common.hlsli:200-205): the guide inputs an application binds from its full-size G-buffer -- IN_VIEWZ, IN_NORMAL_ROUGHNESS,
// IN_MV, the confidence / disocclusion-mix / base-colour inputs -- are read at rectOrigin + pixelPos; the kernels get a view of the
// texture that starts at rectOrigin.  Noisy signals, outputs and pool textures are addressed at pixelPos itself.
Surf WithRectOrigin(Surf s, ResourceType type, const Texture& t, const CommonSettings& cs)
{
    const uint32_t ox = cs.rectOrigin[0], oy = cs.rectOrigin[1];
    if (!ox && !oy) return s;
    switch (type)
    {
        case ResourceType::IN_VIEWZ:
        case ResourceType::IN_NORMAL_ROUGHNESS:
        case ResourceType::IN_MV:
        case ResourceType::IN_DIFF_CONFIDENCE:
        case ResourceType::IN_SPEC_CONFIDENCE:
        case ResourceType::IN_DISOCCLUSION_THRESHOLD_MIX:
        case ResourceType::IN_BASECOLOR_METALNESS: break;
        default: return s;
    }
    s.base += (size_t)oy * s.pitch + (size_t)ox * BytesPerTexel(t.format);
    s.w -= (int)ox;
    s.h -= (int)oy;
    s.y1 -= (int)oy;
    s.lrows -= oy;
    return s;
}

// Roughness table: every function of the 10-bit roughness code alone that the REBLUR spatial filters need, evaluated with the
// host libm in the reference's operation order (Common.hlsli:311-317 GetSpecMagicCurve, NRD.hlsli:520-523
// _REBLUR_GetHitDistanceNormalization, NRD.hlsli:386-392 _NRD_GetSpecularDominantFactor).  `volatile` keeps every intermediate a
// rounded float (no contraction, no excess precision), so the entries are what a plain IEEE evaluation of the HLSL gives.
Result UpdateRoughnessLut(NrdCudaContext* ctx, const float* hitDistParams, cudaStream_t stream)
{
    if (ctx->lutValid && ctx->lutKey[0] == hitDistParams[2] && ctx->lutKey[1] == hitDistParams[3]) return Result::SUCCESS;
    if (!ctx->roughnessLut || !ctx->roughnessLutStaging) return Fail(ctx, Result::FAILURE, "roughness table was not allocated");
    if (ctx->lutValid) cudaEventSynchronize(ctx->lutUploaded); // the previous upload has left the staging buffer
    float* table = ctx->roughnessLutStaging;
    for (int i = 0; i < 1024; i++)
    {
        volatile float r = (float)i / 1023.0f;
        volatile float rr = r * r;
        volatile float e0 = exp2f(-200.0f * rr);
        volatile float f = 1.0f - e0;
        volatile float pw = powf(r, 0.25f); // Pow01: r is already in [0, 1]
        volatile float smc = f * pw;
        // p.w * roughness * roughness: left to right
        volatile float t0 = hitDistParams[3] * r;
        volatile float t1 = t0 * r;
        volatile float e1 = exp2f(t1);
        float sat = e1 > 0.0f ? (e1 < 1.0f ? e1 : 1.0f) : 0.0f;
        volatile float d = (hitDistParams[2] - 1.0f) * sat;
        volatile float hitK = 1.0f + d;
        volatile float la = 39.0029f * r;
        volatile float lb = 39.4115f - la;
        volatile float aLog = 0.298475f * logf(lb);
        table[i * 4 + 0] = smc;
        table[i * 4 + 1] = hitK;
        table[i * 4 + 2] = aLog;
        table[i * 4 + 3] = r;
    }
    cudaError_t e = cudaMemcpyAsync(ctx->roughnessLut, table, 1024 * 4 * sizeof(float), cudaMemcpyHostToDevice, stream);
    if (e == cudaSuccess) e = cudaEventRecord(ctx->lutUploaded, stream);
    if (e != cudaSuccess) return Fail(ctx, Result::FAILURE, std::string("roughness table upload: ") + cudaGetErrorString(e));
    ctx->lutKey[0] = hitDistParams[2];
    ctx->lutKey[1] = hitDistParams[3];
    ctx->lutValid = true;
    return Result::SUCCESS;
}

// Loads every kernel the instance's pipelines map to (see NRD_B200_LAUNCH): nothing may be loaded lazily once barriers spin.
void PreloadKernels(const NrdCudaContext* ctx, cudaError_t (*launchPass)(const PassLaunch&))
{
    alignas(16) static unsigned char dummy[1024] = {}; // a zeroed constant block big enough for every denoiser
    ((RelaxConstants*)dummy)->gDiffCheckerboard = ((RelaxConstants*)dummy)->gSpecCheckerboard = 2; // (checkerboard off; in preload mode every variant is loaded anyway)
    const Scheduler& scheduler = *(const Scheduler*)ctx->instance;
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
    if (((volatile unsigned*)a.flags)[kMaxPeers] != 0) return; // an earlier barrier of this context timed out: do not wait 2 s per pass again
    const unsigned long long start = GlobalTimerNs();
    while ((int)(*mine - a.epoch) < 0)
    {
        if ((long long)(GlobalTimerNs() - start) > a.timeout)
        {
            a.flags[kMaxPeers] = a.epoch; // sticky error word (device side) ...
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
// With `fused` the block that finishes last also runs the inter-GPU barrier of this pass (one launch instead of two): every
// block fences its stores system-wide before it takes a ticket, the holder of the last ticket fences again and signals.
__global__ void __launch_bounds__(256) GhostPushKernel(const __grid_constant__ PushArgs a, const __grid_constant__ BarrierArgs b, int fused)
{
    const PushItem& it = a.items[blockIdx.y];
    const uint4* src = (const uint4*)it.src;
    uint4* dst = (uint4*)it.dst;
    const size_t n = it.bytes / 16;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) dst[i] = src[i];
    if (!fused) return;
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
} // namespace nrdb200

namespace
{
// The executor's own kernels are preloaded like the pass kernels (NRD_B200_LAUNCH): the stand-alone barrier is first needed by a
// pass that pushes nothing, i.e. possibly while this rank's previous (fused) barrier still spins for a peer whose launches the host
// has not issued yet -- a lazy load at that point would wait for the spinning kernel.
void PreloadExecutorKernels()
{
    cudaFuncAttributes fa;
    (void)cudaFuncGetAttributes(&fa, nrdb200::ClearKernel);
    (void)cudaFuncGetAttributes(&fa, nrdb200::StripBarrierKernel);
    (void)cudaFuncGetAttributes(&fa, nrdb200::GhostPushKernel);
}

BarrierArgs NextBarrier(NrdCudaContext* ctx)
{
    BarrierArgs a{};
    a.flags = (unsigned*)ctx->arena;
    for (uint32_t i = 0; i < ctx->world; i++) a.delta[i] = ctx->peerDelta[i];
    a.rank = ctx->rank;
    a.world = ctx->world;
    a.epoch = ++ctx->epoch;
    a.timeout = kBarrierTimeoutNs;
    a.hostError = ctx->hostError;
    return a;
}

Result Barrier(NrdCudaContext* ctx, cudaStream_t stream)
{
    if (!StripMode(ctx) || ctx->world <= 1) return Result::SUCCESS;
    const BarrierArgs a = NextBarrier(ctx);
    StripBarrierKernel<<<1, 32, 0, stream>>>(a);
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? Result::SUCCESS : Fail(ctx, Result::FAILURE, std::string("strip barrier: ") + cudaGetErrorString(e));
}

// Sends the boundary rows of `textures` (arena-owned, just written by this rank) to the ghost rows of the two neighbours and
// then meets all ranks (the barrier rides on the last push launch; without anything to push it is a launch of its own).
Result PushGhostsAndBarrier(NrdCudaContext* ctx, const Texture* const* textures, uint32_t n, cudaStream_t stream)
{
    if (!StripMode(ctx) || ctx->world <= 1) return Result::SUCCESS;
    if (ctx->halo == 0 || n == 0) return Barrier(ctx, stream);
    PushArgs a{};
    uint32_t items = 0;
    unsigned long long maxBytes = 0;
    bool barrierDone = false;
    auto flush = [&](bool fuse) -> Result {
        if (!items) return Result::SUCCESS;
        unsigned blocksX = (unsigned)((maxBytes / 16 + 256 * 8 - 1) / (256 * 8)); // ~8 x 16 B per thread
        if (blocksX < 1) blocksX = 1;
        if (blocksX > kSmCount * 4) blocksX = kSmCount * 4;
        BarrierArgs b{};
        if (fuse) b = NextBarrier(ctx), barrierDone = true;
        GhostPushKernel<<<dim3(blocksX, items), 256, 0, stream>>>(a, b, fuse ? 1 : 0);
        cudaError_t e = cudaGetLastError();
        items = 0;
        maxBytes = 0;
        return e == cudaSuccess ? Result::SUCCESS : Fail(ctx, Result::FAILURE, std::string("ghost push: ") + cudaGetErrorString(e));
    };
    for (uint32_t i = 0; i < n; i++)
    {
        const Texture& t = *textures[i];
        if (!t.owned || !t.rows || !t.haloRows) continue;
        const uint32_t H = t.haloRows, cnt = t.rows < H ? t.rows : H; // ConnectPeers guarantees rows >= H except for the last strip
        uint8_t* base = (uint8_t*)t.ptr;
        if (ctx->rank > 0)
        {
            // my first rows are the bottom ghost rows of the strip above: they follow its own rows, i.e. local rows [H + rowsAbove, ...) there
            const uint32_t rowsAbove = (ctx->stripStart[ctx->rank] - ctx->stripStart[ctx->rank - 1]) / t.downsample;
            a.items[items++] = {base + (size_t)H * t.pitch, base + ctx->peerDelta[ctx->rank - 1] + (size_t)(H + rowsAbove) * t.pitch, (unsigned long long)cnt * t.pitch};
            if ((unsigned long long)cnt * t.pitch > maxBytes) maxBytes = (unsigned long long)cnt * t.pitch;
        }
        if (ctx->rank + 1 < ctx->world)
        {
            // my last rows are the top ghost rows of the strip below: local rows [H - cnt, H) over there
            a.items[items++] = {base + (size_t)(H + t.rows - cnt) * t.pitch, base + ctx->peerDelta[ctx->rank + 1] + (size_t)(H - cnt) * t.pitch, (unsigned long long)cnt * t.pitch};
            if ((unsigned long long)cnt * t.pitch > maxBytes) maxBytes = (unsigned long long)cnt * t.pitch;
        }
        if (items + 2 > (uint32_t)kMaxPushItems)
        {
            Result r = flush(false);
            if (r != Result::SUCCESS) return r;
        }
    }
    Result r = flush(true);
    if (r != Result::SUCCESS) return r;
    return barrierDone ? Result::SUCCESS : Barrier(ctx, stream);
}
} // namespace

extern "C" {

NRD_API Result nrdCudaCreateContext(Instance* instance, const NrdCudaContextDesc* desc, NrdCudaContext** out)
{
    if (!instance || !desc || !out) return Result::INVALID_ARGUMENT;
    if (!desc->resourceWidth || !desc->resourceHeight || desc->stripY1 < desc->stripY0 || desc->stripY1 > desc->resourceHeight) return Result::INVALID_ARGUMENT;
    if (desc->stripHeight == 0 && (desc->stripY0 != 0 || desc->stripY1 != desc->resourceHeight)) return Result::INVALID_ARGUMENT;
    if (desc->stripHeight != 0)
    {
        // uniform strips of whole 16-row tiles; the last ranks may own fewer (or no) rows
        if (desc->stripHeight % 16 != 0 || desc->stripY0 % 16 != 0 || desc->stripY1 - desc->stripY0 > desc->stripHeight) return Result::INVALID_ARGUMENT;
        if (desc->stripY1 != desc->resourceHeight && desc->stripY1 % 16 != 0) return Result::INVALID_ARGUMENT;
    }
    int deviceCount = 0;
    if (cudaGetDeviceCount(&deviceCount) != cudaSuccess || deviceCount == 0) return Result::FAILURE; // no silent CPU path: fail loudly
    if (cudaSetDevice(desc->device) != cudaSuccess) return Result::FAILURE;

    NrdCudaContext* ctx = new NrdCudaContext();
    ctx->instance = instance;
    ctx->desc = *desc;
    if (desc->stripHeight != 0)
    {
        // ghost rows: whole tiles, at most one strip (they are refreshed by the direct neighbours only)
        // at least one tile: the kernels read the centre pixel's fixed neighbourhoods (up to +-4 rows, REBLUR history fix up to
        // +-14) without an owner lookup (device/common.cuh Near)
        ctx->halo = ((uint32_t)desc->haloRows + 15u) / 16u * 16u;
        if (ctx->halo < 16u) ctx->halo = 16u;
        if (ctx->halo > desc->stripHeight) ctx->halo = desc->stripHeight;
    }
    const InstanceDesc& id = GetInstanceDesc(*instance);
    ctx->permanent.resize(id.permanentPoolSize);
    ctx->transient.resize(id.transientPoolSize);
    for (uint32_t i = 0; i < id.permanentPoolSize; i++) DescribeTexture(ctx, id.permanentPool[i].format, id.permanentPool[i].downsampleFactor, ctx->permanent[i]);
    for (uint32_t i = 0; i < id.transientPoolSize; i++) DescribeTexture(ctx, id.transientPool[i].format, id.transientPool[i].downsampleFactor, ctx->transient[i]);
    if (StripMode(ctx))
    {
        // foreign device pointers cannot be reached by the peers: the strips of the IN_* / OUT_* textures live in the arena too
        for (uint32_t t = 0; t < (uint32_t)ResourceType::MAX_NUM; t++)
        {
            Format f;
            if (ExpectedUserFormat((ResourceType)t, f, ((Scheduler*)instance)->HasDenoiser(Denoiser::SIGMA_SHADOW_TRANSLUCENCY))) DescribeTexture(ctx, f, 1, ctx->user[t]);
        }
    }
    // one arena, identical layout on every rank
    size_t offset = kArenaHeader;
    auto place = [&](Texture& t) {
        if (!t.owned) return;
        t.ptr = (void*)offset;
        offset += (t.pitch * t.allocRows + 255) & ~(size_t)255;
    };
    DescribeTexture(ctx, Format::RGBA32_SFLOAT, 1, ctx->guide);
    for (Texture& t : ctx->permanent) place(t);
    for (Texture& t : ctx->transient) place(t);
    for (Texture& t : ctx->user) place(t);
    place(ctx->guide);
    ctx->arenaBytes = offset;
    cudaError_t e = cudaMalloc((void**)&ctx->arena, ctx->arenaBytes);
    if (e != cudaSuccess)
    {
        delete ctx;
        return Result::FAILURE;
    }
    if (cudaMalloc((void**)&ctx->roughnessLut, 1024 * 4 * sizeof(float)) != cudaSuccess || cudaMallocHost((void**)&ctx->roughnessLutStaging, 1024 * 4 * sizeof(float)) != cudaSuccess ||
        cudaEventCreateWithFlags(&ctx->lutUploaded, cudaEventDisableTiming) != cudaSuccess)
    {
        nrdCudaDestroyContext(ctx);
        return Result::FAILURE;
    }
    if (StripMode(ctx))
    {
        if (cudaHostAlloc((void**)&ctx->hostError, sizeof(unsigned), cudaHostAllocMapped | cudaHostAllocPortable) != cudaSuccess)
        {
            nrdCudaDestroyContext(ctx);
            return Result::FAILURE;
        }
        *ctx->hostError = 0;
    }
    cudaMemset(ctx->arena, 0, ctx->arenaBytes);
    // the memset runs on the legacy default stream, the context is used on the caller's (non-blocking) streams and by peers:
    // nothing may touch the arena (barrier flags included) before it is zero
    cudaDeviceSynchronize();
    auto rebase = [&](Texture& t) {
        if (t.owned) t.ptr = ctx->arena + (size_t)t.ptr;
    };
    for (Texture& t : ctx->permanent) rebase(t);
    for (Texture& t : ctx->transient) rebase(t);
    for (Texture& t : ctx->user) rebase(t);
    rebase(ctx->guide);
    *out = ctx;
    return Result::SUCCESS;
}

NRD_API void nrdCudaDestroyContext(NrdCudaContext* ctx)
{
    if (!ctx) return;
    cudaSetDevice(ctx->desc.device);
    cudaDeviceSynchronize();
    for (int i = 0; i < kMaxPeers; i++)
        if (ctx->peerOpened[i]) cudaIpcCloseMemHandle(ctx->peerArena[i]);
    if (ctx->peerSlot >= 0)
    {
        std::lock_guard<std::mutex> lock(g_slotMutex);
        g_slotUsed[ctx->peerSlot] = false;
    }
    if (ctx->arena) cudaFree(ctx->arena);
    if (ctx->roughnessLut) cudaFree(ctx->roughnessLut);
    if (ctx->roughnessLutStaging) cudaFreeHost(ctx->roughnessLutStaging);
    if (ctx->lutUploaded) cudaEventDestroy(ctx->lutUploaded);
    if (ctx->hostError) cudaFreeHost(ctx->hostError);
    for (ForeignTexture& f : ctx->foreign)
        if (f.shadow) cudaFree(f.shadow);
    for (cudaEvent_t ev : ctx->timingEvents)
        if (ev) cudaEventDestroy(ev);
    delete ctx;
}

NRD_API Result nrdCudaSetUserTexture(NrdCudaContext* ctx, uint32_t resourceType, void* devicePtr, size_t pitchBytes, uint32_t format)
{
    if (!ctx || resourceType >= (uint32_t)ResourceType::TRANSIENT_POOL || format >= (uint32_t)Format::MAX_NUM) return Result::INVALID_ARGUMENT;
    if (StripMode(ctx)) return Fail(ctx, Result::UNSUPPORTED, "strip mode: user textures live in the context's arena, fill them through nrdCudaGetTexture / nrdCudaCopyTexture");
    Format expected;
    if (!ExpectedUserFormat((ResourceType)resourceType, expected, ((Scheduler*)ctx->instance)->HasDenoiser(Denoiser::SIGMA_SHADOW_TRANSLUCENCY)))
        return Fail(ctx, Result::UNSUPPORTED, "resource type not consumed by the supported denoisers");
    ForeignTexture& foreign = ctx->foreign[resourceType];
    const bool wider = (Format)format != expected;
    if (wider)
    {
        // a wider format of the same kind: bind a shadow texture in the kernels' format, converted around the passes
        FormatInfo have, want;
        const bool packedNormals = expected == Format::R10_G10_B10_A2_UNORM; // the normal encoding is a property of the library build (LibraryDesc)
        if (packedNormals || !ConvertibleFormat((Format)format, have) || !ConvertibleFormat(expected, want) ||
            (have.channels < want.channels && (ResourceType)resourceType != ResourceType::IN_MV) || (want.kind != 0 && have.kind == 0))
            return Fail(ctx, Result::UNSUPPORTED, "unsupported format for this resource type (see nrd_b200.h: the listed format, or a 16- / 32-bit float format with at least its channels)");
    }
    if (foreign.shadow) cudaFree(foreign.shadow); // (the previous binding of this resource type is replaced from here on)
    foreign = ForeignTexture{};
    if (wider)
    {
        const size_t shadowPitch = ((size_t)ctx->desc.resourceWidth * BytesPerTexel(expected) + 255) & ~(size_t)255;
        if (cudaMalloc(&foreign.shadow, shadowPitch * ctx->desc.resourceHeight) != cudaSuccess)
        {
            foreign.shadow = nullptr;
            ctx->user[resourceType] = Texture{};
            return Fail(ctx, Result::FAILURE, "cudaMalloc of the format-conversion shadow texture failed");
        }
        cudaMemset(foreign.shadow, 0, shadowPitch * ctx->desc.resourceHeight);
        foreign.ptr = devicePtr;
        foreign.pitch = pitchBytes;
        foreign.format = (Format)format;
        devicePtr = foreign.shadow;
        pitchBytes = shadowPitch;
        format = (uint32_t)expected;
    }
    Texture& t = ctx->user[resourceType];
    t.ptr = devicePtr;
    t.pitch = pitchBytes;
    t.format = (Format)format;
    t.downsample = 1;
    t.width = ctx->desc.resourceWidth;
    t.height = ctx->desc.resourceHeight;
    OwnedRows(ctx->desc, 1, t.height, t.firstRow, t.rows);
    t.allocRows = t.rows;
    t.owned = false;
    return Result::SUCCESS;
}

NRD_API Result nrdCudaGetTexture(NrdCudaContext* ctx, uint32_t resourceType, uint32_t indexInPool, NrdCudaTextureInfo* info)
{
    if (!ctx || !info) return Result::INVALID_ARGUMENT;
    const Texture* t = Resolve(ctx, (ResourceType)resourceType, indexInPool);
    if (!t) return Result::INVALID_ARGUMENT;
    info->devicePtr = t->OwnPtr();
    info->pitchBytes = t->pitch;
    info->format = (uint32_t)t->format;
    info->width = t->width;
    info->height = t->height;
    info->firstRow = t->firstRow;
    info->rowsNum = t->rows;
    return Result::SUCCESS;
}

NRD_API Result nrdCudaGetArena(NrdCudaContext* ctx, void** devicePtr, size_t* bytes)
{
    if (!ctx || !devicePtr || !bytes) return Result::INVALID_ARGUMENT;
    *devicePtr = ctx->arena;
    *bytes = ctx->arenaBytes;
    return Result::SUCCESS;
}

NRD_API Result nrdCudaGetIpcHandle(NrdCudaContext* ctx, void* handleOut)
{
    static_assert(sizeof(cudaIpcMemHandle_t) == NRD_CUDA_IPC_HANDLE_SIZE, "IPC handle size");
    if (!ctx || !handleOut) return Result::INVALID_ARGUMENT;
    if (!StripMode(ctx)) return Fail(ctx, Result::UNSUPPORTED, "not a strip-mode context");
    cudaIpcMemHandle_t h;
    cudaError_t e = cudaIpcGetMemHandle(&h, ctx->arena);
    if (e != cudaSuccess) return Fail(ctx, Result::FAILURE, std::string("cudaIpcGetMemHandle: ") + cudaGetErrorString(e));
    memcpy(handleOut, &h, sizeof(h));
    return Result::SUCCESS;
}

NRD_API Result nrdCudaConnectPeers(NrdCudaContext* ctx, uint32_t rank, uint32_t worldSize, const void* ipcHandles, void* const* arenas, const uint16_t* stripStarts)
{
    if (!ctx || worldSize == 0 || worldSize > (uint32_t)kMaxPeers || rank >= worldSize || (!ipcHandles == !arenas)) return Result::INVALID_ARGUMENT;
    if (!StripMode(ctx)) return Fail(ctx, Result::UNSUPPORTED, "not a strip-mode context");
    if (ctx->connected) return Fail(ctx, Result::FAILURE, "peers already connected");
    // strip starts: given explicitly (cost-aware partition) or uniform strips of stripHeight rows
    for (uint32_t i = 0; i <= worldSize; i++)
    {
        uint32_t y = stripStarts ? stripStarts[i] : i * (uint32_t)ctx->desc.stripHeight;
        if (!stripStarts && (i == worldSize || y > ctx->desc.resourceHeight)) y = ctx->desc.resourceHeight;
        ctx->stripStart[i] = y;
    }
    if (ctx->stripStart[0] != 0 || ctx->stripStart[worldSize] != ctx->desc.resourceHeight) return Fail(ctx, Result::INVALID_ARGUMENT, "the strips do not cover the frame");
    for (uint32_t i = 0; i < worldSize; i++)
    {
        const uint32_t rows = ctx->stripStart[i + 1] - ctx->stripStart[i];
        if (ctx->stripStart[i + 1] <= ctx->stripStart[i] || ctx->stripStart[i] % 16 != 0 || rows > ctx->desc.stripHeight)
            return Fail(ctx, Result::INVALID_ARGUMENT, "every strip must start on a multiple of 16, own rows and fit stripHeight");
        if (rows < ctx->halo && i + 1 < worldSize) return Fail(ctx, Result::INVALID_ARGUMENT, "haloRows exceeds the height of a strip (ghost rows are refreshed by the direct neighbours only)");
    }
    if (ctx->stripStart[rank] != ctx->desc.stripY0 || ctx->stripStart[rank + 1] != ctx->desc.stripY1) return Fail(ctx, Result::INVALID_ARGUMENT, "stripY0/stripY1 do not match the strip table");
    cudaSetDevice(ctx->desc.device);
    for (uint32_t i = 0; i < worldSize; i++)
    {
        if (i == rank) { ctx->peerArena[i] = ctx->arena; continue; }
        if (arenas) ctx->peerArena[i] = arenas[i];
        else
        {
            cudaIpcMemHandle_t h;
            memcpy(&h, (const uint8_t*)ipcHandles + (size_t)i * sizeof(h), sizeof(h));
            cudaError_t e = cudaIpcOpenMemHandle(&ctx->peerArena[i], h, cudaIpcMemLazyEnablePeerAccess);
            if (e != cudaSuccess) return Fail(ctx, Result::FAILURE, std::string("cudaIpcOpenMemHandle: ") + cudaGetErrorString(e));
            ctx->peerOpened[i] = true;
        }
    }
    for (uint32_t i = 0; i < (uint32_t)kMaxPeers; i++) ctx->peerDelta[i] = i < worldSize ? (long long)((uint8_t*)ctx->peerArena[i] - ctx->arena) : 0;
    {
        std::lock_guard<std::mutex> lock(g_slotMutex);
        for (int s = 0; s < kMaxPeerSlots && ctx->peerSlot < 0; s++)
            if (!g_slotUsed[s]) { g_slotUsed[s] = true; ctx->peerSlot = s; }
    }
    if (ctx->peerSlot < 0) return Fail(ctx, Result::FAILURE, "too many strip-mode contexts in one process");
    PeerTable table{};
    for (uint32_t i = 0; i < (uint32_t)kMaxPeers; i++) table.delta[i] = ctx->peerDelta[i];
    for (uint32_t i = 0; i <= (uint32_t)kMaxPeers; i++) table.start[i] = i <= worldSize ? (int)ctx->stripStart[i] : 0x7fffffff;
    if (worldSize < (uint32_t)kMaxPeers) table.start[worldSize] = 0x7fffffff; // rows >= start[world] do not exist: never counted as an owner change
    cudaError_t e = SetPeerTables(ctx->peerSlot, &table);
    if (e != cudaSuccess) return Fail(ctx, Result::FAILURE, std::string("peer table: ") + cudaGetErrorString(e));
    ctx->rank = rank;
    ctx->world = worldSize;
    ctx->connected = true;
    PreloadKernels(ctx, worldSize > 1 ? nrdb200::LaunchPass : nrdb200_single::LaunchPass);
    PreloadExecutorKernels();
    return Result::SUCCESS;
}

}  // extern "C"

namespace
{
// converts one user texture that is bound in a wider format between the application's copy and the shadow the kernels use
Result ConvertForeign(NrdCudaContext* ctx, uint32_t type, bool toNative, cudaStream_t stream)
{
    const ForeignTexture& f = ctx->foreign[type];
    if (!f.shadow) return Result::SUCCESS;
    const Texture& t = ctx->user[type];
    FormatInfo app, native;
    ConvertibleFormat(f.format, app);
    ConvertibleFormat(t.format, native);
    ConvertArgs a{};
    a.width = t.width;
    a.height = t.height;
    if (toNative)
    {
        a.src = (const uint8_t*)f.ptr; a.srcPitch = f.pitch; a.srcChannels = app.channels; a.srcKind = app.kind;
        a.dst = (uint8_t*)t.ptr; a.dstPitch = t.pitch; a.dstChannels = native.channels; a.dstKind = native.kind;
    }
    else
    {
        a.src = (const uint8_t*)t.ptr; a.srcPitch = t.pitch; a.srcChannels = native.channels; a.srcKind = native.kind;
        a.dst = (uint8_t*)f.ptr; a.dstPitch = f.pitch; a.dstChannels = app.channels; a.dstKind = app.kind;
    }
    ConvertFormatKernel<<<dim3((a.width + 31) / 32, (a.height + 7) / 8), dim3(32, 8), 0, stream>>>(a);
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? Result::SUCCESS : Fail(ctx, Result::FAILURE, std::string("format conversion: ") + cudaGetErrorString(e));
}
Result ConvertForeignAll(NrdCudaContext* ctx, bool inputs, cudaStream_t stream)
{
    for (uint32_t t = 0; t < (uint32_t)ResourceType::MAX_NUM; t++)
    {
        if (!ctx->foreign[t].shadow) continue;
        const char* name = GetResourceTypeString((ResourceType)t);
        if (!name || (strncmp(name, "IN_", 3) == 0) != inputs) continue;
        const Result r = ConvertForeign(ctx, t, inputs, stream);
        if (r != Result::SUCCESS) return r;
    }
    return Result::SUCCESS;
}

// pushMask: bit i set = the ghost rows of resource i must be refreshed after this pass (it is read by a later pass)
Result ExecuteInternal(NrdCudaContext* ctx, const DispatchDesc* d, void* stream, uint32_t pushMask)
{
    if (!ctx || !d) return Result::INVALID_ARGUMENT;
    if (ctx->hostError && *(volatile unsigned*)ctx->hostError)
        return Fail(ctx, Result::FAILURE, "a strip barrier of this context timed out waiting for a peer (epoch " + std::to_string(*(volatile unsigned*)ctx->hostError) + "): its outputs since then are not valid");
    const InstanceDesc& id = GetInstanceDesc(*ctx->instance);
    if (d->pipelineIndex >= id.pipelinesNum) return Result::INVALID_ARGUMENT;
    const char* shader = id.pipelines[d->pipelineIndex].shaderFileName;
    const PassKind kind = ((Scheduler*)ctx->instance)->PipelineKind(d->pipelineIndex);
    const CommonSettings& cs = ((Scheduler*)ctx->instance)->Common();
    // Dynamic resolution (Source/InstanceImpl.cpp:834-856, Shaders/Include/Common.hlsli:200-222): the passes run over rectSize <= resourceSize;
    // the application's guide inputs are addressed at rectOrigin + pixel (WithRectOrigin), everything else at the pixel itself.
    if (cs.resourceSize[0] != ctx->desc.resourceWidth || cs.resourceSize[1] != ctx->desc.resourceHeight)
        return Fail(ctx, Result::INVALID_ARGUMENT, "CommonSettings::resourceSize differs from the size the context was created for");
    if (cs.rectOrigin[0] + (uint32_t)cs.rectSize[0] > cs.resourceSize[0] || cs.rectOrigin[1] + (uint32_t)cs.rectSize[1] > cs.resourceSize[1])
        return Fail(ctx, Result::INVALID_ARGUMENT, "rectOrigin + rectSize exceeds resourceSize");
    const bool subRect = cs.rectSize[0] != cs.resourceSize[0] || cs.rectSize[1] != cs.resourceSize[1] || cs.rectOrigin[0] || cs.rectOrigin[1];
    if (subRect && StripMode(ctx) && ctx->world > 1)
        return Fail(ctx, Result::UNSUPPORTED, "dynamic resolution (rectSize != resourceSize) is not implemented for multi-GPU strips");
    if (StripMode(ctx) && !ctx->connected && (ctx->desc.stripY0 != 0 || ctx->desc.stripY1 != ctx->desc.resourceHeight))
        return Fail(ctx, Result::FAILURE, "strip-mode context used before nrdCudaConnectPeers");

    PassLaunch p{};
    p.kind = kind;
    p.constants = d->constantBufferData;
    p.constantsSize = d->constantBufferDataSize;
    p.texNum = d->resourcesNum;
    p.gridW = d->gridWidth;
    p.gridH = d->gridHeight;
    p.stream = (cudaStream_t)stream;
    if (d->resourcesNum > 32) return Fail(ctx, Result::FAILURE, "too many resources in one dispatch");
    for (uint32_t i = 0; i < d->resourcesNum; i++)
    {
        const ResourceDesc& r = d->resources[i];
        const Texture* t = Resolve(ctx, r.type, r.indexInPool);
        if (!t) return Fail(ctx, Result::INVALID_ARGUMENT, std::string("unbound resource ") + GetResourceTypeString(r.type) + " for " + d->name);
        p.tex[i] = WithRectOrigin(ToSurf(ctx, *t), r.type, *t, cs);
        p.texBytes[i] = (uint8_t)BytesPerTexel(t->format);
    }
    // checkerboarded REBLUR inputs (ReblurSettings::checkerboardMode) bind the same passes: the pre-pass resolves them, temporal
    // accumulation slows down on resolved pixels; RELAX and the split-screen passes reject them in their launchers
    // decoded-guide surface: ClassifyTiles (first pass of every REBLUR frame) fills it, all later passes of the frame read it
    const bool isReblur = kind.family == Family::REBLUR, isRelax = kind.family == Family::RELAX, isClear = kind.family == Family::CLEAR;
    const bool buildsGuide = (isReblur || isRelax) && kind.pass == Pass::ClassifyTiles;
    const bool isSplitScreen = kind.pass == Pass::SplitScreen; // may be the only pass of the frame (splitScreen >= 1)
    const bool readsGuide = (isReblur || isRelax) && !buildsGuide && !isSplitScreen; // every other REBLUR / RELAX pass reads it (REBLUR: and the roughness table)
    p.guide = ToSurf(ctx, ctx->guide);
    if (buildsGuide)
    {
        const Texture* nr = Resolve(ctx, ResourceType::IN_NORMAL_ROUGHNESS, 0);
        if (!nr) return Fail(ctx, Result::INVALID_ARGUMENT, "unbound resource IN_NORMAL_ROUGHNESS for ClassifyTiles (it also builds the guide surface)");
        p.guideNr = WithRectOrigin(ToSurf(ctx, *nr), ResourceType::IN_NORMAL_ROUGHNESS, *nr, cs);
        p.guideMode = 1;
    }
    else if (readsGuide)
    {
        if (!ctx->guideValid) return Fail(ctx, Result::FAILURE, std::string(shader) + " dispatched before ClassifyTiles of the same frame");
        if (isReblur)
        {
            ReblurConstants rc;
            memcpy(&rc, d->constantBufferData, sizeof(rc));
            Result lr = UpdateRoughnessLut(ctx, rc.gHitDistParams, (cudaStream_t)stream);
            if (lr != Result::SUCCESS) return lr;
            p.roughnessLut = ctx->roughnessLut;
        }
        p.guideMode = 2;
    }
    // rows to produce: the context's strip (the full frame on one GPU)
    p.rowBegin = ctx->desc.stripY0;
    p.rowEnd = ctx->desc.stripY1;
    if (subRect)
    {
        // dynamic resolution: no pass produces rows beyond max(rect, previous rect) (the grids of USE_MAX_DIMS passes), whole tiles
        const uint32_t rows = ((uint32_t)std::max(cs.rectSize[1], cs.rectSizePrev[1]) + 15u) & ~15u;
        p.rowEnd = (int)std::min<uint32_t>((uint32_t)p.rowEnd, rows);
    }
    {
        // profiling aid (one GPU only): NRD_B200_DEBUG_ROWS="y0,y1" restricts every pass to a row range, to cost a strip in isolation
        static const char* dbg = getenv("NRD_B200_DEBUG_ROWS");
        int a = 0, b = 0;
        if (dbg && !StripMode(ctx) && sscanf(dbg, "%d,%d", &a, &b) == 2 && a % 16 == 0 && b > a && b <= (int)ctx->desc.resourceHeight) p.rowBegin = a, p.rowEnd = b;
    }

    // NRD_B200_FORCE_STRIP_KERNELS: run a one-GPU context on the strip build of the kernels.  The two builds are compiled
    // separately and differ in the last bits (FMA contraction); N-GPU results are bit-identical to THIS configuration.
    const bool stripBuild = (StripMode(ctx) && ctx->world > 1) || getenv("NRD_B200_FORCE_STRIP_KERNELS") != nullptr;
    cudaError_t e;
    const bool timed = ctx->timing && ctx->timingCount < 64 && !isClear;
    const uint32_t slot = ctx->timingCount;
    const Texture* clearTarget = isClear && d->resourcesNum ? Resolve(ctx, d->resources[0].type, d->resources[0].indexInPool) : nullptr;
    if (clearTarget && !clearTarget->owned)
    {
        // an application texture (IN_MV / OUT_* are storage outputs of some passes): its pitch may exceed the row and the bytes
        // between rows are not ours -- clear exactly width x height texels
        e = clearTarget->rows ? cudaMemset2DAsync(clearTarget->ptr, clearTarget->pitch, 0, (size_t)clearTarget->width * BytesPerTexel(clearTarget->format), clearTarget->rows,
                                                  (cudaStream_t)stream)
                              : cudaSuccess;
    }
    else if (isClear)
        e = LaunchClear(p);
    else
    {
        if (timed) cudaEventRecord(ctx->timingEvents[3 * slot + 0], p.stream);
        e = stripBuild ? nrdb200::LaunchPass(p) : nrdb200_single::LaunchPass(p);
        if (timed) cudaEventRecord(ctx->timingEvents[3 * slot + 1], p.stream);
    }

    if (e == cudaErrorNotSupported) return Fail(ctx, Result::UNSUPPORTED, std::string("no CUDA kernel for pass ") + shader);
    if (e != cudaSuccess) return Fail(ctx, Result::FAILURE, std::string(shader) + ": " + cudaGetErrorString(e));
    g_launchCount.fetch_add(1, std::memory_order_relaxed);
    if (buildsGuide) ctx->guideValid = true;
    const Texture* list[33];
    uint32_t n = 0;
    if (!isClear && pushMask) // clears zero the ghost rows locally
    {
        for (uint32_t i = 0; i < d->resourcesNum; i++)
            if ((pushMask >> i) & 1u) list[n++] = Resolve(ctx, d->resources[i].type, d->resources[i].indexInPool);
    }
    // (the guide surface needs no push: ClassifyTiles decodes its ghost rows from the ghost rows of the inputs, which arrived with the
    // frame-start push; the barrier below still separates it from the neighbours' far taps, which load the guide from its owner)
    const Result pr = PushGhostsAndBarrier(ctx, list, n, p.stream);
    if (timed)
    {
        cudaEventRecord(ctx->timingEvents[3 * slot + 2], p.stream);
        ctx->timingCount = slot + 1;
    }
    return pr;
}

uint32_t StorageMask(const DispatchDesc* d)
{
    uint32_t m = 0;
    for (uint32_t i = 0; i < d->resourcesNum && i < 32; i++)
        if (d->resources[i].descriptorType == DescriptorType::STORAGE_TEXTURE) m |= 1u << i;
    return m;
}

// frame start: the IN_* strips the application just wrote are pushed to the neighbours' ghost rows, then all ranks meet
Result FrameStart(NrdCudaContext* ctx, void* stream)
{
    if (StripMode(ctx) && ctx->world > 1)
    {
        const Texture* list[(size_t)ResourceType::MAX_NUM];
        uint32_t n = 0;
        for (uint32_t t = 0; t < (uint32_t)ResourceType::MAX_NUM; t++)
        {
            const char* name = GetResourceTypeString((ResourceType)t);
            if (ctx->user[t].ptr && name && !strncmp(name, "IN_", 3)) list[n++] = &ctx->user[t];
        }
        return PushGhostsAndBarrier(ctx, list, n, (cudaStream_t)stream);
    }
    return Barrier(ctx, (cudaStream_t)stream);
}
} // namespace

extern "C" {

NRD_API Result nrdCudaExecuteDispatch(NrdCudaContext* ctx, const DispatchDesc* d, void* stream)
{
    if (!ctx || !d) return Result::INVALID_ARGUMENT;
    // textures bound in a wider format: convert what this pass reads before it and what it writes after it (nrdCudaDenoise does it per frame)
    for (uint32_t i = 0; i < d->resourcesNum; i++)
        if (d->resources[i].descriptorType == DescriptorType::TEXTURE && (uint32_t)d->resources[i].type < (uint32_t)ResourceType::TRANSIENT_POOL)
        {
            const Result cr = ConvertForeign(ctx, (uint32_t)d->resources[i].type, true, (cudaStream_t)stream);
            if (cr != Result::SUCCESS) return cr;
        }
    const Result r = ExecuteInternal(ctx, d, stream, StorageMask(d)); // no look-ahead here: refresh the ghosts of every output
    if (r != Result::SUCCESS) return r;
    for (uint32_t i = 0; i < d->resourcesNum; i++)
        if (d->resources[i].descriptorType == DescriptorType::STORAGE_TEXTURE && (uint32_t)d->resources[i].type < (uint32_t)ResourceType::TRANSIENT_POOL)
        {
            const Result cr = ConvertForeign(ctx, (uint32_t)d->resources[i].type, false, (cudaStream_t)stream);
            if (cr != Result::SUCCESS) return cr;
        }
    return Result::SUCCESS;
}

NRD_API Result nrdCudaDenoise(NrdCudaContext* ctx, const Identifier* identifiers, uint32_t identifiersNum, void* stream, uint32_t* launches)
{
    if (!ctx) return Result::INVALID_ARGUMENT;
    const DispatchDesc* dispatches = nullptr;
    uint32_t n = 0;
    Result r = GetComputeDispatches(*ctx->instance, identifiers, identifiersNum, dispatches, n);
    if (r != Result::SUCCESS) return r;
    r = ConvertForeignAll(ctx, true, (cudaStream_t)stream); // inputs bound in a wider format -> the kernels' format
    if (r != Result::SUCCESS) return r;
    r = FrameStart(ctx, stream);
    if (r != Result::SUCCESS) return r;
    for (uint32_t i = 0; i < n; i++)
    {
        // an output needs fresh ghost rows only if a later pass reads it before anyone overwrites it; what survives the frame
        // may be read next frame unless it is transient
        uint32_t mask = 0;
        const DispatchDesc& d = dispatches[i];
        for (uint32_t k = 0; k < d.resourcesNum && k < 32; k++)
        {
            const ResourceDesc& out = d.resources[k];
            if (out.descriptorType != DescriptorType::STORAGE_TEXTURE) continue;
            bool decided = false, needed = false;
            for (uint32_t j = i + 1; j < n && !decided; j++)
                for (uint32_t m = 0; m < dispatches[j].resourcesNum && !decided; m++)
                {
                    const ResourceDesc& use = dispatches[j].resources[m];
                    if (use.type != out.type || use.indexInPool != out.indexInPool) continue;
                    decided = true;
                    needed = use.descriptorType == DescriptorType::TEXTURE;
                    // a pass may bind a texture both ways (never in the supported chains); reading wins
                    for (uint32_t q = m + 1; q < dispatches[j].resourcesNum; q++)
                        if (dispatches[j].resources[q].type == out.type && dispatches[j].resources[q].indexInPool == out.indexInPool &&
                            dispatches[j].resources[q].descriptorType == DescriptorType::TEXTURE)
                            needed = true;
                }
            if (!decided) needed = out.type != ResourceType::TRANSIENT_POOL; // history, or an output a denoiser re-reads next frame (SIGMA)
            if (needed) mask |= 1u << k;
        }
        r = ExecuteInternal(ctx, &d, stream, mask);
        if (r != Result::SUCCESS) return r;
    }
    r = ConvertForeignAll(ctx, false, (cudaStream_t)stream); // outputs -> the application's wider format
    if (r != Result::SUCCESS) return r;
    if (launches) *launches = n;
    return Result::SUCCESS;
}

NRD_API Result nrdCudaUploadTexture(NrdCudaContext* ctx, uint32_t resourceType, uint32_t indexInPool, const void* hostPtr, size_t hostPitchBytes)
{
    if (!ctx || !hostPtr) return Result::INVALID_ARGUMENT;
    const Texture* t = Resolve(ctx, (ResourceType)resourceType, indexInPool);
    if (!t) return Result::INVALID_ARGUMENT;
    if (!t->rows) return Result::SUCCESS;
    cudaError_t e = cudaMemcpy2D(t->OwnPtr(), t->pitch, hostPtr, hostPitchBytes, (size_t)t->width * BytesPerTexel(t->format), t->rows, cudaMemcpyHostToDevice);
    return e == cudaSuccess ? Result::SUCCESS : Fail(ctx, Result::FAILURE, cudaGetErrorString(e));
}

NRD_API Result nrdCudaDownloadTexture(NrdCudaContext* ctx, uint32_t resourceType, uint32_t indexInPool, void* hostPtr, size_t hostPitchBytes)
{
    if (!ctx || !hostPtr) return Result::INVALID_ARGUMENT;
    const Texture* t = Resolve(ctx, (ResourceType)resourceType, indexInPool);
    if (!t) return Result::INVALID_ARGUMENT;
    if (!t->rows) return Result::SUCCESS;
    cudaError_t e = cudaMemcpy2D(hostPtr, hostPitchBytes, t->OwnPtr(), t->pitch, (size_t)t->width * BytesPerTexel(t->format), t->rows, cudaMemcpyDeviceToHost);
    return e == cudaSuccess ? Result::SUCCESS : Fail(ctx, Result::FAILURE, cudaGetErrorString(e));
}

NRD_API Result nrdCudaCopyTexture(NrdCudaContext* ctx, uint32_t resourceType, uint32_t indexInPool, void* ptr, size_t pitchBytes, int32_t toContext, void* stream)
{
    if (!ctx || !ptr) return Result::INVALID_ARGUMENT;
    const Texture* t = Resolve(ctx, (ResourceType)resourceType, indexInPool);
    if (!t) return Result::INVALID_ARGUMENT;
    if (!t->rows) return Result::SUCCESS;
    const size_t rowBytes = (size_t)t->width * BytesPerTexel(t->format);
    cudaError_t e = toContext ? cudaMemcpy2DAsync(t->OwnPtr(), t->pitch, ptr, pitchBytes, rowBytes, t->rows, cudaMemcpyDefault, (cudaStream_t)stream)
                              : cudaMemcpy2DAsync(ptr, pitchBytes, t->OwnPtr(), t->pitch, rowBytes, t->rows, cudaMemcpyDefault, (cudaStream_t)stream);
    return e == cudaSuccess ? Result::SUCCESS : Fail(ctx, Result::FAILURE, cudaGetErrorString(e));
}

NRD_API Result nrdCudaBarrier(NrdCudaContext* ctx, void* stream)
{
    if (!ctx) return Result::INVALID_ARGUMENT;
    return FrameStart(ctx, stream);
}

NRD_API Result nrdCudaSynchronize(NrdCudaContext* ctx, void* stream)
{
    if (!ctx) return Result::INVALID_ARGUMENT;
    cudaError_t e = cudaStreamSynchronize((cudaStream_t)stream);
    if (e != cudaSuccess) return Fail(ctx, Result::FAILURE, std::string("cudaStreamSynchronize: ") + cudaGetErrorString(e));
    if (StripMode(ctx) && ctx->world > 1)
    {
        unsigned err = 0;
        e = cudaMemcpy(&err, ctx->arena + sizeof(unsigned) * kMaxPeers, sizeof(err), cudaMemcpyDeviceToHost);
        if (e != cudaSuccess) return Fail(ctx, Result::FAILURE, cudaGetErrorString(e));
        if (err) return Fail(ctx, Result::FAILURE, "strip barrier timed out waiting for a peer (epoch " + std::to_string(err) + ")");
    }
    return Result::SUCCESS;
}

NRD_API Result nrdCudaSetTiming(NrdCudaContext* ctx, int32_t enable)
{
    if (!ctx) return Result::INVALID_ARGUMENT;
    if (enable && !ctx->timingEvents[0])
        for (cudaEvent_t& ev : ctx->timingEvents)
            if (cudaEventCreate(&ev) != cudaSuccess) return Fail(ctx, Result::FAILURE, "cudaEventCreate failed");
    ctx->timing = enable != 0;
    ctx->timingCount = 0;
    return Result::SUCCESS;
}

NRD_API Result nrdCudaGetTiming(NrdCudaContext* ctx, float* kernelMs, float* exchangeMs, uint32_t capacity, uint32_t* count)
{
    if (!ctx || !count) return Result::INVALID_ARGUMENT;
    const uint32_t n = ctx->timingCount < capacity ? ctx->timingCount : capacity;
    for (uint32_t i = 0; i < n; i++)
    {
        float k = 0.0f, x = 0.0f;
        if (cudaEventSynchronize(ctx->timingEvents[3 * i + 2]) != cudaSuccess || cudaEventElapsedTime(&k, ctx->timingEvents[3 * i], ctx->timingEvents[3 * i + 1]) != cudaSuccess ||
            cudaEventElapsedTime(&x, ctx->timingEvents[3 * i + 1], ctx->timingEvents[3 * i + 2]) != cudaSuccess)
            return Fail(ctx, Result::FAILURE, "timing events are not complete");
        if (kernelMs) kernelMs[i] = k;
        if (exchangeMs) exchangeMs[i] = x;
    }
    *count = n;
    ctx->timingCount = 0;
    return Result::SUCCESS;
}

NRD_API const char* nrdCudaGetLastError(NrdCudaContext* ctx) { return ctx ? ctx->lastError.c_str() : ""; }
NRD_API uint64_t nrdCudaGetLaunchCount() { return g_launchCount.load(); }
}
