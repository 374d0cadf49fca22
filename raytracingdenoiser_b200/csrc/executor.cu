// CUDA executor: owns the pool textures in HBM and turns DispatchDesc[] into sm_90a kernel launches.
// Takes the role of the reference's optional NRI integration layer (Integration/NRDIntegration.hpp: pool creation
// :292-363, Denoise :516-623, Dispatch :625-803).  Stream order replaces the SRV/UAV barriers (:667-704); constants
// travel as __grid_constant__ kernel parameters instead of a constant-buffer ring (:721-749).
// Where the textures live and how strips of a multi-GPU run exchange rows and meet between passes: arena.h.
#include "arena.h"
#include "device/launch.h"
#include "constants.h"
#include "scheduler.h"

#include <atomic>
#include <cstdio>
#include <cstring>
#include <iterator>
#include <string>
#include <vector>

using namespace nrd;
using namespace nrdb200;

namespace
{
std::atomic<uint64_t> g_launchCount{0};

// The user textures the supported denoisers read or write, with the one format the kernels are written for.
struct UserTexture
{
    ResourceType type;
    Format format;
    bool isInput;          // written by the application before the frame (IN_*), else written by the passes (OUT_*)
    bool readAtRectOrigin; // WithRectOrigin (Common.hlsli:200-205): a guide input an application binds from its full-size G-buffer
};
constexpr UserTexture kUserTextures[] = {
    {ResourceType::IN_MV, Format::RGBA16_SFLOAT, true, true},
    {ResourceType::IN_NORMAL_ROUGHNESS, Format::R10_G10_B10_A2_UNORM, true, true},
    {ResourceType::IN_VIEWZ, Format::R32_SFLOAT, true, true},
    // optional inputs (CommonSettings::isHistoryConfidenceAvailable / isDisocclusionThresholdMixAvailable / isBaseColorMetalnessAvailable)
    {ResourceType::IN_DIFF_CONFIDENCE, Format::R8_UNORM, true, true},
    {ResourceType::IN_SPEC_CONFIDENCE, Format::R8_UNORM, true, true},
    {ResourceType::IN_DISOCCLUSION_THRESHOLD_MIX, Format::R8_UNORM, true, true},
    {ResourceType::IN_BASECOLOR_METALNESS, Format::RGBA8_UNORM, true, true},
    {ResourceType::IN_DIFF_RADIANCE_HITDIST, Format::RGBA16_SFLOAT, true, false},
    {ResourceType::IN_SPEC_RADIANCE_HITDIST, Format::RGBA16_SFLOAT, true, false},
    {ResourceType::IN_PENUMBRA, Format::R16_SFLOAT, true, false},
    {ResourceType::IN_TRANSLUCENCY, Format::RGBA8_UNORM, true, false},
    {ResourceType::IN_SIGNAL, Format::RGBA16_SFLOAT, true, false}, // REFERENCE denoiser
    {ResourceType::OUT_DIFF_RADIANCE_HITDIST, Format::RGBA16_SFLOAT, false, false},
    {ResourceType::OUT_SPEC_RADIANCE_HITDIST, Format::RGBA16_SFLOAT, false, false},
    {ResourceType::OUT_SHADOW_TRANSLUCENCY, Format::R8_UNORM, false, false},
    {ResourceType::OUT_SIGNAL, Format::RGBA16_SFLOAT, false, false}, // REFERENCE denoiser
};
constexpr UserTexture kTranslucentShadow = {ResourceType::OUT_SHADOW_TRANSLUCENCY, Format::RGBA8_UNORM, false, false};

// nullptr for a resource type no supported denoiser reads or writes.  OUT_SHADOW_TRANSLUCENCY is R8 for SIGMA_SHADOW and
// RGBA8 for SIGMA_SHADOW_TRANSLUCENCY: `translucent` picks.
const UserTexture* FindUserTexture(ResourceType type, bool translucent = false)
{
    if (type == ResourceType::OUT_SHADOW_TRANSLUCENCY && translucent) return &kTranslucentShadow;
    for (const UserTexture& u : kUserTextures)
        if (u.type == type) return &u;
    return nullptr;
}

bool Translucent(const Instance* instance) { return ((const Scheduler*)instance)->HasDenoiser(Denoiser::SIGMA_SHADOW_TRANSLUCENCY); }
} // namespace

// ---- user textures in a format above the minimum (Include/NRDDescs.h:43-137 lists MINIMUM formats) -----------------------------------
// The kernels are written for one format per user texture (kUserTextures).  A texture bound in a wider format of the same kind
// (e.g. RGBA32_SFLOAT radiance, R16_SFLOAT viewZ, RG16_SFLOAT motion) gets a shadow copy in the kernels' format: inputs are converted
// into it before the passes that read them, outputs out of it after the passes that wrote them (one streaming kernel per texture).
// Accepted (WiderFormat): at least the channels (IN_MV excepted: a two-channel motion vector has no z), no UNORM source for a
// float format, never for the packed normals (their encoding is a property of the library build, LibraryDesc).
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
bool WiderFormat(ResourceType type, Format have, Format want)
{
    FormatInfo h, w;
    if (want == Format::R10_G10_B10_A2_UNORM || !ConvertibleFormat(have, h) || !ConvertibleFormat(want, w)) return false;
    return (h.channels >= w.channels || type == ResourceType::IN_MV) && (w.kind == 0 || h.kind != 0);
}
struct ConvertSide
{
    uint8_t* texels;
    size_t pitch;
    int channels, kind, bytes; // bytes per texel
};
ConvertSide Side(void* texels, size_t pitch, Format f)
{
    FormatInfo info{};
    ConvertibleFormat(f, info);
    return {(uint8_t*)texels, pitch, info.channels, info.kind, (int)BytesPerTexel(f)};
}
struct ConvertArgs
{
    ConvertSide src, dst;
    int width, height;
};
// channels the source does not have read 0 (a two-channel motion vector has no z / w), extra source channels are dropped
__global__ void __launch_bounds__(256) ConvertFormatKernel(const __grid_constant__ ConvertArgs a)
{
    const int x = blockIdx.x * 32 + threadIdx.x, y = blockIdx.y * 8 + threadIdx.y;
    if (x >= a.width || y >= a.height) return;
    const uint8_t* s = a.src.texels + (size_t)y * a.src.pitch + (size_t)x * a.src.bytes;
    uint8_t* d = a.dst.texels + (size_t)y * a.dst.pitch + (size_t)x * a.dst.bytes;
    for (int ch = 0; ch < a.dst.channels; ch++) StoreChannel(d, a.dst.kind, ch, ch < a.src.channels ? LoadChannel(s, a.src.kind, ch) : 0.0f);
}
// The application's texture behind a shadow: a device pointer bound in a wider format (nrdCudaSetUserTexture), or a CUDA array
// in any accepted format (nrdCudaSetUserTextureArray; converted by the kernels of device/user_arrays.cu).
struct ForeignTexture
{
    void* ptr = nullptr;     // pointer binding: the application's texture
    size_t pitch = 0;
    bool isArray = false;    // array binding: the application's CUDA array, through a surface object created at bind time
    cudaSurfaceObject_t surface = 0;
    Format format = Format::R8_UNORM;
    void* shadow = nullptr;  // cudaMalloc'ed copy in the kernels' format (NrdCudaContext::user[] points at it)
};
TexelFormat TexelFormatOf(Format f)
{
    FormatInfo info{};
    ConvertibleFormat(f, info);
    return {info.channels, info.kind, (int)BytesPerTexel(f)};
}
void ReleaseForeign(ForeignTexture& f)
{
    // an array binding always has a shadow: cudaFree waits for the device, so no conversion still uses the surface below
    if (f.shadow) cudaFree(f.shadow);
    if (f.isArray) cudaDestroySurfaceObject(f.surface);
    f = ForeignTexture{};
}

struct NrdCudaContext
{
    Instance* instance = nullptr;
    Arena arena; // the context description, the textures' memory and the strip exchange
    std::vector<Texture> permanent, transient;
    Texture user[(size_t)ResourceType::MAX_NUM];
    ForeignTexture foreign[(size_t)ResourceType::MAX_NUM]; // user textures bound in a wider format than the kernels' (see ConvertFormatKernel)
    // decoded-guide surface of the REBLUR spatial passes (surf.h PassLaunch::guide): written by ClassifyTiles, the first pass
    // of every REBLUR frame, read by PrePass / Blur / PostBlur of the same frame
    Texture guide;
    bool guideValid = false;
    // strip mode: a copy of every guide input (UserTexture::readAtRectOrigin) in the arena, bound instead of the input on frames
    // that stage (StagesInputs); FrameStart fills it and records for which rectOrigin
    Texture staged[(size_t)ResourceType::MAX_NUM];
    bool stagedFrame = false;
    uint32_t stagedOrigin[2] = {0, 0};
    bool repartitioned = false; // nrdCudaRepartition ran since the last frame start: no dispatch before the next one
    // roughness table of the REBLUR spatial passes (surf.h PassLaunch::roughnessLut), rebuilt when hitDistanceParameters change
    float* roughnessLut = nullptr;     // device, 1024 x float4 (allocated with the context: no cudaMalloc -- an implicit device
    float* roughnessLutStaging = nullptr; // synchronisation -- may happen while a strip barrier spins); pinned staging copy
    cudaEvent_t lutUploaded = nullptr;
    // NRD_B200_FORCE_STRIP_KERNELS at creation: run a one-GPU context on the strip build of the kernels.  The two builds are
    // compiled separately and differ in the last bits (FMA contraction); N-GPU results are bit-identical to THIS configuration.
    bool forceStripKernels = false;
    bool timing = false;                  // nrdCudaSetTiming: three events per dispatch (before the kernel, after it, after push + barrier)
    cudaEvent_t timingEvents[3 * 64] = {};
    uint32_t timingCount = 0;
    float lutKey[2] = {0.0f, 0.0f};
    bool lutValid = false;
    std::string lastError;
};

namespace
{
// the refusal of both user-texture bindings on a strip-mode context
constexpr const char* kStripUserTextures = "strip mode: user textures live in the context's arena, fill them through nrdCudaGetTexture / nrdCudaCopyTexture";

Result Fail(NrdCudaContext* ctx, Result r, const std::string& msg)
{
    if (ctx) ctx->lastError = msg;
    return r;
}

const Texture* Resolve(NrdCudaContext* ctx, ResourceType type, uint32_t index)
{
    if (type == ResourceType::PERMANENT_POOL) return index < ctx->permanent.size() ? &ctx->permanent[index] : nullptr;
    if (type == ResourceType::TRANSIENT_POOL) return index < ctx->transient.size() ? &ctx->transient[index] : nullptr;
    if ((uint32_t)type < (uint32_t)ResourceType::MAX_NUM && ctx->user[(uint32_t)type].ptr) return &ctx->user[(uint32_t)type];
    return nullptr;
}

// The guide inputs (UserTexture::readAtRectOrigin) are read at rectOrigin + pixelPos: the kernels get a view of the texture that
// starts at rectOrigin.  Noisy signals, outputs and pool textures are addressed at pixelPos itself.
Surf WithRectOrigin(Surf s, ResourceType type, const Texture& t, const CommonSettings& cs)
{
    const uint32_t ox = cs.rectOrigin[0], oy = cs.rectOrigin[1];
    const UserTexture* u = FindUserTexture(type);
    if ((!ox && !oy) || !u || !u->readAtRectOrigin) return s;
    s.base += (size_t)oy * s.pitch + (size_t)ox * BytesPerTexel(t.format);
    s.w -= (int)ox;
    s.h -= (int)oy;
    s.y1 -= (int)oy;
    s.lrows -= oy;
    return s;
}

// Connected strips cannot take that view when rectOrigin.y != 0: shifted by whole rows, a strip's own and ghost rows would hold
// rows of other strips (the kernels' Near() loads skip the owner lookup).  They stage the guide inputs instead: FrameStart
// gathers each into a copy with the view's rows in the strip's rows (GatherRectOriginKernel), the passes bind that copy.
bool StagesInputs(const NrdCudaContext* ctx, const CommonSettings& cs) { return ctx->arena.strip.MultiGpu() && cs.rectOrigin[1] != 0; }

// the guide inputs this frame's passes bind: the optional ones only with their CommonSettings flag (recipes_*.cpp bind a dummy otherwise)
bool GuideInputRead(ResourceType type, const CommonSettings& cs)
{
    switch (type)
    {
        case ResourceType::IN_DIFF_CONFIDENCE:
        case ResourceType::IN_SPEC_CONFIDENCE: return cs.isHistoryConfidenceAvailable;
        case ResourceType::IN_DISOCCLUSION_THRESHOLD_MIX: return cs.isDisocclusionThresholdMixAvailable;
        case ResourceType::IN_BASECOLOR_METALNESS: return cs.isBaseColorMetalnessAvailable;
        default: return true;
    }
}

// the staged copy as the passes see it: origin 0, and the size of the one-GPU view, so that every clamp is the same
Surf StagedView(const NrdCudaContext* ctx, ResourceType type, const CommonSettings& cs)
{
    Surf s = ctx->arena.ToSurf(ctx->staged[(uint32_t)type]);
    s.w -= (int)cs.rectOrigin[0];
    s.h -= (int)cs.rectOrigin[1];
    return s;
}

// the rect must fit the textures the context was created for
Result CheckRect(NrdCudaContext* ctx, const CommonSettings& cs)
{
    const NrdCudaContextDesc& desc = ctx->arena.desc;
    if (cs.resourceSize[0] != desc.resourceWidth || cs.resourceSize[1] != desc.resourceHeight)
        return Fail(ctx, Result::INVALID_ARGUMENT, "CommonSettings::resourceSize differs from the size the context was created for");
    if (cs.rectOrigin[0] + (uint32_t)cs.rectSize[0] > cs.resourceSize[0] || cs.rectOrigin[1] + (uint32_t)cs.rectSize[1] > cs.resourceSize[1])
        return Fail(ctx, Result::INVALID_ARGUMENT, "rectOrigin + rectSize exceeds resourceSize");
    return Result::SUCCESS;
}

// every texture the arena holds, in placement order: one arena, identical layout on every rank
std::vector<Texture*> ArenaTextures(NrdCudaContext* ctx)
{
    std::vector<Texture*> placed;
    for (std::vector<Texture>* pool : {&ctx->permanent, &ctx->transient})
        for (Texture& t : *pool) placed.push_back(&t);
    for (Texture& t : ctx->user) placed.push_back(&t);
    placed.push_back(&ctx->guide);
    // the staged guide inputs (StagesInputs): the arena is mapped by the peers once, so they are carved out of it too, after
    // everything else
    for (const UserTexture& u : kUserTextures)
        if (ctx->staged[(uint32_t)u.type].owned) placed.push_back(&ctx->staged[(uint32_t)u.type]);
    return placed;
}

// nrdCudaSetTiming: a slot of three events, like a dispatch (before the kernel, after it, after the exchange); nullptr when full / off
cudaEvent_t* TimingSlot(NrdCudaContext* ctx) { return ctx->timing && ctx->timingCount < 64 ? &ctx->timingEvents[3 * ctx->timingCount++] : nullptr; }

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

// a zeroed shadow of user texture `type` in the kernels' format (ForeignTexture::shadow); on failure the type is left unbound
Result AllocateShadow(NrdCudaContext* ctx, uint32_t type, Format format, size_t& pitch)
{
    ForeignTexture& f = ctx->foreign[type];
    pitch = ((size_t)ctx->arena.desc.resourceWidth * BytesPerTexel(format) + 255) & ~(size_t)255;
    if (cudaMalloc(&f.shadow, pitch * ctx->arena.desc.resourceHeight) != cudaSuccess)
    {
        f.shadow = nullptr;
        ctx->user[type] = Texture{};
        return Fail(ctx, Result::FAILURE, "cudaMalloc of the format-conversion shadow texture failed");
    }
    cudaMemset(f.shadow, 0, pitch * ctx->arena.desc.resourceHeight);
    return Result::SUCCESS;
}

// The user textures in `types` (bit i = ResourceType i) that are bound as CUDA arrays, converted in one launch: array -> shadow
// (toShadow) or shadow -> array, the whole resourceSize.  Pointer bindings are ConvertForeign's.
Result ConvertArrays(NrdCudaContext* ctx, uint64_t types, bool toShadow, cudaStream_t stream)
{
    static_assert(std::size(kUserTextures) <= (size_t)kMaxArrayCopies && (size_t)ResourceType::MAX_NUM <= 64, "one launch, one bit per type");
    ArrayCopyArgs a{};
    for (const UserTexture& u : kUserTextures)
    {
        const ForeignTexture& f = ctx->foreign[(uint32_t)u.type];
        if (!f.isArray || !((types >> (uint32_t)u.type) & 1u)) continue;
        const Texture& t = ctx->user[(uint32_t)u.type];
        a.items[a.n++] = {f.surface, (uint8_t*)t.ptr, t.pitch, TexelFormatOf(f.format), TexelFormatOf(t.format), (int)t.width, (int)t.height};
    }
    if (!a.n) return Result::SUCCESS;
    // a one-GPU context that runs the strip build of the kernels (NRD_B200_FORCE_STRIP_KERNELS) runs its conversions there too
    const cudaError_t e = ctx->forceStripKernels ? nrdb200::LaunchArrayCopies(a, toShadow, stream) : nrdb200_single::LaunchArrayCopies(a, toShadow, stream);
    return e == cudaSuccess ? Result::SUCCESS : Fail(ctx, Result::FAILURE, std::string("CUDA array conversion: ") + cudaGetErrorString(e));
}

uint64_t Bit(ResourceType type) { return 1ull << (uint32_t)type; }

// REBLUR / RELAX ClassifyTiles, the first pass of every frame, also decodes the guide surface from IN_NORMAL_ROUGHNESS, which
// the dispatch does not bind (surf.h PassLaunch::guideNr)
bool BuildsGuide(const PassKind& kind) { return (kind.family == Family::REBLUR || kind.family == Family::RELAX) && kind.pass == Pass::ClassifyTiles; }

// the user textures some dispatch of `d[0, n)` binds as `binding`
uint64_t TypesBoundAs(const DispatchDesc* d, uint32_t n, DescriptorType binding)
{
    uint64_t types = 0;
    for (uint32_t i = 0; i < n; i++)
        for (uint32_t j = 0; j < d[i].resourcesNum; j++)
            if (d[i].resources[j].descriptorType == binding && FindUserTexture(d[i].resources[j].type)) types |= Bit(d[i].resources[j].type);
    return types;
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
    ctx->forceStripKernels = getenv("NRD_B200_FORCE_STRIP_KERNELS") != nullptr;
    Arena& arena = ctx->arena;
    arena.desc = *desc;
    if (desc->stripHeight != 0)
    {
        // ghost rows: whole tiles, at most one strip (they are refreshed by the direct neighbours only)
        // at least one tile: the kernels read the centre pixel's fixed neighbourhoods (up to +-4 rows, REBLUR history fix up to
        // +-14) without an owner lookup (device/common.cuh Near)
        arena.strip.halo = ((uint32_t)desc->haloRows + 15u) / 16u * 16u;
        if (arena.strip.halo < 16u) arena.strip.halo = 16u;
        if (arena.strip.halo > desc->stripHeight) arena.strip.halo = desc->stripHeight;
    }
    const InstanceDesc& id = GetInstanceDesc(*instance);
    for (uint32_t i = 0; i < id.permanentPoolSize; i++) ctx->permanent.push_back(arena.Describe(id.permanentPool[i].format, id.permanentPool[i].downsampleFactor, true));
    for (uint32_t i = 0; i < id.transientPoolSize; i++) ctx->transient.push_back(arena.Describe(id.transientPool[i].format, id.transientPool[i].downsampleFactor, true));
    // foreign device pointers cannot be reached by the peers: in strip mode the strips of the user textures live in the arena too
    if (arena.StripMode())
        for (const UserTexture& u : kUserTextures) ctx->user[(uint32_t)u.type] = arena.Describe(FindUserTexture(u.type, Translucent(instance))->format, 1, true);
    ctx->guide = arena.Describe(Format::RGBA32_SFLOAT, 1, true);
    if (arena.StripMode())
        for (const UserTexture& u : kUserTextures)
            if (u.readAtRectOrigin) ctx->staged[(uint32_t)u.type] = arena.Describe(u.format, 1, true);
    const std::vector<Texture*> placed = ArenaTextures(ctx);
    if (arena.Allocate(placed.data(), placed.size()) != Result::SUCCESS || cudaMalloc((void**)&ctx->roughnessLut, 1024 * 4 * sizeof(float)) != cudaSuccess ||
        cudaMallocHost((void**)&ctx->roughnessLutStaging, 1024 * 4 * sizeof(float)) != cudaSuccess ||
        cudaEventCreateWithFlags(&ctx->lutUploaded, cudaEventDisableTiming) != cudaSuccess)
    {
        nrdCudaDestroyContext(ctx);
        return Result::FAILURE;
    }
    *out = ctx;
    return Result::SUCCESS;
}

NRD_API void nrdCudaDestroyContext(NrdCudaContext* ctx)
{
    if (!ctx) return;
    cudaSetDevice(ctx->arena.desc.device);
    cudaDeviceSynchronize();
    ctx->arena.Release();
    if (ctx->roughnessLut) cudaFree(ctx->roughnessLut);
    if (ctx->roughnessLutStaging) cudaFreeHost(ctx->roughnessLutStaging);
    if (ctx->lutUploaded) cudaEventDestroy(ctx->lutUploaded);
    for (ForeignTexture& f : ctx->foreign) ReleaseForeign(f);
    for (cudaEvent_t ev : ctx->timingEvents)
        if (ev) cudaEventDestroy(ev);
    delete ctx;
}

NRD_API Result nrdCudaSetUserTexture(NrdCudaContext* ctx, uint32_t resourceType, void* devicePtr, size_t pitchBytes, uint32_t format)
{
    if (!ctx || resourceType >= (uint32_t)ResourceType::TRANSIENT_POOL || format >= (uint32_t)Format::MAX_NUM) return Result::INVALID_ARGUMENT;
    if (ctx->arena.StripMode()) return Fail(ctx, Result::UNSUPPORTED, kStripUserTextures);
    const UserTexture* u = FindUserTexture((ResourceType)resourceType, Translucent(ctx->instance));
    if (!u) return Fail(ctx, Result::UNSUPPORTED, "resource type not consumed by the supported denoisers");
    const Format expected = u->format;
    ForeignTexture& foreign = ctx->foreign[resourceType];
    // a wider format of the same kind: bind a shadow texture in the kernels' format, converted around the passes
    const bool wider = (Format)format != expected;
    if (wider && !WiderFormat(u->type, (Format)format, expected))
        return Fail(ctx, Result::UNSUPPORTED, "unsupported format for this resource type (see nrd_b200.h: the listed format, or a 16- / 32-bit float format with at least its channels)");
    ReleaseForeign(foreign); // (the previous binding of this resource type is replaced from here on)
    if (wider)
    {
        size_t shadowPitch = 0;
        const Result r = AllocateShadow(ctx, resourceType, expected, shadowPitch);
        if (r != Result::SUCCESS) return r;
        foreign.ptr = devicePtr;
        foreign.pitch = pitchBytes;
        foreign.format = (Format)format;
        devicePtr = foreign.shadow;
        pitchBytes = shadowPitch;
    }
    ctx->user[resourceType] = ctx->arena.Describe(expected, 1, false, devicePtr, pitchBytes);
    return Result::SUCCESS;
}

NRD_API Result nrdCudaSetUserTextureArray(NrdCudaContext* ctx, uint32_t resourceType, void* cudaArray, uint32_t format)
{
    if (!ctx) return Result::INVALID_ARGUMENT;
    if (!cudaArray) return Fail(ctx, Result::INVALID_ARGUMENT, "the CUDA array is null");
    if (resourceType >= (uint32_t)ResourceType::TRANSIENT_POOL || format >= (uint32_t)Format::MAX_NUM) return Fail(ctx, Result::INVALID_ARGUMENT, "resource type or format out of range");
    if (ctx->arena.StripMode()) return Fail(ctx, Result::UNSUPPORTED, kStripUserTextures);
    const UserTexture* u = FindUserTexture((ResourceType)resourceType, Translucent(ctx->instance));
    if (!u) return Fail(ctx, Result::UNSUPPORTED, "resource type not consumed by the supported denoisers");
    const Format expected = u->format;
    if ((Format)format != expected && !WiderFormat(u->type, (Format)format, expected))
        return Fail(ctx, Result::UNSUPPORTED, "unsupported format for this resource type (see nrd_b200.h: the listed format, or a 16- / 32-bit float format with at least its channels)");
    cudaChannelFormatDesc cd{};
    cudaExtent extent{};
    unsigned flags = 0;
    cudaError_t e = cudaArrayGetInfo(&cd, &extent, &flags, (cudaArray_t)cudaArray);
    if (e != cudaSuccess)
    {
        cudaGetLastError(); // not sticky: keep it from being reported by the next launch check
        return Fail(ctx, Result::INVALID_ARGUMENT, std::string("cudaArrayGetInfo: ") + cudaGetErrorString(e));
    }
    if ((flags & (cudaArrayLayered | cudaArrayCubemap)) || extent.depth != 0)
        return Fail(ctx, Result::UNSUPPORTED, "a layered, cube map or 3D CUDA array: bind a 2D array (level 0 of a mipmapped array)");
    if (!(flags & cudaArraySurfaceLoadStore))
        return Fail(ctx, Result::UNSUPPORTED, "the CUDA array was created without cudaArraySurfaceLoadStore (CUDA_ARRAY3D_SURFACE_LDST): the executor converts it through a surface");
    const uint32_t elementBytes = (uint32_t)(cd.x + cd.y + cd.z + cd.w) / 8;
    if (elementBytes != BytesPerTexel((Format)format))
        return Fail(ctx, Result::UNSUPPORTED, "the CUDA array's element size (" + std::to_string(elementBytes) + " bytes) differs from the bytes per texel of the format (" +
                                                  std::to_string(BytesPerTexel((Format)format)) + ")");
    if (extent.width < ctx->arena.desc.resourceWidth || extent.height < ctx->arena.desc.resourceHeight)
        return Fail(ctx, Result::INVALID_ARGUMENT, "the CUDA array (" + std::to_string(extent.width) + " x " + std::to_string(extent.height) +
                                                       ") is smaller than the context's resource size");
    cudaResourceDesc rd{};
    rd.resType = cudaResourceTypeArray;
    rd.res.array.array = (cudaArray_t)cudaArray;
    cudaSurfaceObject_t surface = 0;
    e = cudaCreateSurfaceObject(&surface, &rd);
    if (e != cudaSuccess)
    {
        cudaGetLastError();
        return Fail(ctx, Result::UNSUPPORTED, std::string("cudaCreateSurfaceObject: ") + cudaGetErrorString(e));
    }
    ForeignTexture& foreign = ctx->foreign[resourceType];
    ReleaseForeign(foreign); // (the previous binding of this resource type is replaced from here on)
    size_t shadowPitch = 0;
    const Result r = AllocateShadow(ctx, resourceType, expected, shadowPitch);
    if (r != Result::SUCCESS)
    {
        cudaDestroySurfaceObject(surface);
        return r;
    }
    foreign.isArray = true;
    foreign.surface = surface;
    foreign.format = (Format)format;
    ctx->user[resourceType] = ctx->arena.Describe(expected, 1, false, foreign.shadow, shadowPitch);
    // the shadow starts as the array: texels no pass writes (outside the rect) go back to the array as the application left them
    return ConvertArrays(ctx, Bit((ResourceType)resourceType), true, nullptr);
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
    *devicePtr = ctx->arena.base;
    *bytes = ctx->arena.bytes;
    return Result::SUCCESS;
}

NRD_API Result nrdCudaGetIpcHandle(NrdCudaContext* ctx, void* handleOut)
{
    static_assert(sizeof(cudaIpcMemHandle_t) == NRD_CUDA_IPC_HANDLE_SIZE, "IPC handle size");
    if (!ctx || !handleOut) return Result::INVALID_ARGUMENT;
    if (!ctx->arena.StripMode()) return Fail(ctx, Result::UNSUPPORTED, "not a strip-mode context");
    cudaIpcMemHandle_t h;
    cudaError_t e = cudaIpcGetMemHandle(&h, ctx->arena.base);
    if (e != cudaSuccess) return Fail(ctx, Result::FAILURE, std::string("cudaIpcGetMemHandle: ") + cudaGetErrorString(e));
    memcpy(handleOut, &h, sizeof(h));
    return Result::SUCCESS;
}

NRD_API Result nrdCudaConnectPeers(NrdCudaContext* ctx, uint32_t rank, uint32_t worldSize, const void* ipcHandles, void* const* arenas, const uint16_t* stripStarts)
{
    if (!ctx) return Result::INVALID_ARGUMENT;
    const Result r = ctx->arena.ConnectPeers(*ctx->instance, rank, worldSize, ipcHandles, arenas, stripStarts, ctx->lastError);
    if (r != Result::SUCCESS || !ctx->arena.strip.MultiGpu()) return r;
    const cudaError_t e = PreloadShiftedCopies(); // the staging kernels run between barriers too
    return e == cudaSuccess ? r : Fail(ctx, Result::FAILURE, std::string("loading the staging kernels: ") + cudaGetErrorString(e));
}

}  // extern "C"

namespace
{
// converts one user texture that is bound in a wider format between the application's copy and the shadow the kernels use
Result ConvertForeign(NrdCudaContext* ctx, ResourceType type, bool toNative, cudaStream_t stream)
{
    const ForeignTexture& f = ctx->foreign[(uint32_t)type];
    if (!f.shadow || f.isArray) return Result::SUCCESS;
    const Texture& t = ctx->user[(uint32_t)type];
    const ConvertSide app = Side(f.ptr, f.pitch, f.format), native = Side(t.ptr, t.pitch, t.format);
    const ConvertArgs a{toNative ? app : native, toNative ? native : app, t.width, t.height};
    ConvertFormatKernel<<<dim3((a.width + 31) / 32, (a.height + 7) / 8), dim3(32, 8), 0, stream>>>(a);
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? Result::SUCCESS : Fail(ctx, Result::FAILURE, std::string("format conversion: ") + cudaGetErrorString(e));
}
Result ConvertForeignAll(NrdCudaContext* ctx, bool inputs, cudaStream_t stream)
{
    for (const UserTexture& u : kUserTextures)
    {
        if (u.isInput != inputs) continue;
        const Result r = ConvertForeign(ctx, u.type, inputs, stream);
        if (r != Result::SUCCESS) return r;
    }
    return Result::SUCCESS;
}

// the user textures a dispatch binds as `binding`: TEXTURE ones to the kernels' format, STORAGE_TEXTURE ones back
Result ConvertBound(NrdCudaContext* ctx, const DispatchDesc* d, DescriptorType binding, cudaStream_t stream)
{
    for (uint32_t i = 0; i < d->resourcesNum; i++)
        if (d->resources[i].descriptorType == binding && FindUserTexture(d->resources[i].type))
        {
            const Result r = ConvertForeign(ctx, d->resources[i].type, binding == DescriptorType::TEXTURE, stream);
            if (r != Result::SUCCESS) return r;
        }
    uint64_t types = TypesBoundAs(d, 1, binding);
    const Scheduler* scheduler = (const Scheduler*)ctx->instance;
    if (binding == DescriptorType::TEXTURE && d->pipelineIndex < GetInstanceDesc(*ctx->instance).pipelinesNum && BuildsGuide(scheduler->PipelineKind(d->pipelineIndex)))
        types |= Bit(ResourceType::IN_NORMAL_ROUGHNESS);
    return ConvertArrays(ctx, types, binding == DescriptorType::TEXTURE, stream);
}

// After the barrier of a pass that wrote staged guide inputs (REBLUR TemporalStabilization with isBaseColorMetalnessAvailable
// patches IN_MV at rectOrigin + pixel): every rank copies its own rows of the input back from the staged view, which it reads
// through the owner lookup, so the application's texture ends the frame as on one GPU.  Texels the pass did not write come back
// unchanged (the gather copied them there).  No barrier follows: the staged rows are next written by the gather of the next
// frame, after the frame-start barrier.
Result PullStaged(NrdCudaContext* ctx, const DispatchDesc* d, const CommonSettings& cs, cudaStream_t stream)
{
    const int ox = (int)cs.rectOrigin[0], oy = (int)cs.rectOrigin[1];
    ShiftedCopyArgs a{};
    a.dx = -ox;
    a.dy = -oy;
    for (uint32_t i = 0; i < d->resourcesNum && a.n < kMaxShiftedCopies; i++)
    {
        const ResourceType type = d->resources[i].type;
        if (d->resources[i].descriptorType != DescriptorType::STORAGE_TEXTURE || !ctx->staged[(uint32_t)type].ptr) continue;
        const Texture& t = ctx->user[(uint32_t)type];
        a.items[a.n++] = {ctx->arena.ToSurf(t), ctx->arena.ToSurf(ctx->staged[(uint32_t)type]), ox, (int)t.width, std::max((int)t.firstRow, oy),
                          (int)t.firstRow + (int)t.rows, (int)BytesPerTexel(t.format)};
    }
    if (!a.n) return Result::SUCCESS;
    cudaEvent_t* ev = TimingSlot(ctx);
    if (ev) cudaEventRecord(ev[0], stream);
    const cudaError_t e = LaunchShiftedCopies(a, true, stream);
    if (ev) cudaEventRecord(ev[1], stream), cudaEventRecord(ev[2], stream);
    return e == cudaSuccess ? Result::SUCCESS : Fail(ctx, Result::FAILURE, std::string("staged input pull: ") + cudaGetErrorString(e));
}

// pushMask: bit i set = the ghost rows of resource i must be refreshed after this pass (it is read by a later pass)
Result ExecuteInternal(NrdCudaContext* ctx, const DispatchDesc* d, void* stream, uint32_t pushMask)
{
    if (!ctx || !d) return Result::INVALID_ARGUMENT;
    const NrdCudaContextDesc& desc = ctx->arena.desc;
    const StripState& strip = ctx->arena.strip;
    if (strip.hostError && *(volatile unsigned*)strip.hostError)
        return Fail(ctx, Result::FAILURE, "a strip barrier of this context timed out waiting for a peer (epoch " + std::to_string(*(volatile unsigned*)strip.hostError) + "): its outputs since then are not valid");
    const InstanceDesc& id = GetInstanceDesc(*ctx->instance);
    if (d->pipelineIndex >= id.pipelinesNum) return Result::INVALID_ARGUMENT;
    const char* shader = id.pipelines[d->pipelineIndex].shaderFileName;
    const PassKind kind = ((Scheduler*)ctx->instance)->PipelineKind(d->pipelineIndex);
    const CommonSettings& cs = ((Scheduler*)ctx->instance)->Common();
    // Dynamic resolution (Source/InstanceImpl.cpp:834-856, Shaders/Include/Common.hlsli:200-222): the passes run over rectSize <= resourceSize;
    // the application's guide inputs are addressed at rectOrigin + pixel (WithRectOrigin, or their staged copies), everything else at
    // the pixel itself.
    const Result rr = CheckRect(ctx, cs);
    if (rr != Result::SUCCESS) return rr;
    const bool subRect = cs.rectSize[0] != cs.resourceSize[0] || cs.rectSize[1] != cs.resourceSize[1] || cs.rectOrigin[0] || cs.rectOrigin[1];
    if (ctx->arena.StripMode() && !strip.connected && (desc.stripY0 != 0 || desc.stripY1 != desc.resourceHeight))
        return Fail(ctx, Result::FAILURE, "strip-mode context used before nrdCudaConnectPeers");
    if (ctx->repartitioned)
        return Fail(ctx, Result::FAILURE, "dispatched after nrdCudaRepartition without a frame start: call nrdCudaBarrier (or nrdCudaDenoise) first");
    const bool staged = StagesInputs(ctx, cs);
    if (staged != ctx->stagedFrame || (staged && (cs.rectOrigin[0] != ctx->stagedOrigin[0] || cs.rectOrigin[1] != ctx->stagedOrigin[1])))
        return Fail(ctx, Result::INVALID_ARGUMENT, "rectOrigin differs from the one of the frame start: call nrdCudaBarrier after SetCommonSettings (strips stage the guide inputs there)");

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
        if (kind.family == Family::CLEAR) p.tex[i] = ctx->arena.ToSurf(*t); // a clear zeroes the whole texture, whatever the rect
        else if (staged && ctx->staged[(uint32_t)r.type].ptr) p.tex[i] = StagedView(ctx, r.type, cs);
        else p.tex[i] = WithRectOrigin(ctx->arena.ToSurf(*t), r.type, *t, cs);
        p.texBytes[i] = (uint8_t)BytesPerTexel(t->format);
    }
    // checkerboarded REBLUR inputs (ReblurSettings::checkerboardMode) bind the same passes: the pre-pass resolves them, temporal
    // accumulation slows down on resolved pixels; RELAX and the split-screen passes reject them in their launchers
    // decoded-guide surface: ClassifyTiles (first pass of every REBLUR frame) fills it, all later passes of the frame read it
    const bool isReblur = kind.family == Family::REBLUR, isRelax = kind.family == Family::RELAX, isClear = kind.family == Family::CLEAR;
    const bool buildsGuide = BuildsGuide(kind);
    const bool isSplitScreen = kind.pass == Pass::SplitScreen; // may be the only pass of the frame (splitScreen >= 1)
    const bool readsGuide = (isReblur || isRelax) && !buildsGuide && !isSplitScreen; // every other REBLUR / RELAX pass reads it (REBLUR: and the roughness table)
    p.guide = ctx->arena.ToSurf(ctx->guide);
    if (buildsGuide)
    {
        const Texture* nr = Resolve(ctx, ResourceType::IN_NORMAL_ROUGHNESS, 0);
        if (!nr) return Fail(ctx, Result::INVALID_ARGUMENT, "unbound resource IN_NORMAL_ROUGHNESS for ClassifyTiles (it also builds the guide surface)");
        p.guideNr = staged ? StagedView(ctx, ResourceType::IN_NORMAL_ROUGHNESS, cs) : WithRectOrigin(ctx->arena.ToSurf(*nr), ResourceType::IN_NORMAL_ROUGHNESS, *nr, cs);
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
    p.rowBegin = desc.stripY0;
    p.rowEnd = desc.stripY1;
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
        if (dbg && !ctx->arena.StripMode() && sscanf(dbg, "%d,%d", &a, &b) == 2 && a % 16 == 0 && b > a && b <= (int)desc.resourceHeight) p.rowBegin = a, p.rowEnd = b;
    }

    const bool stripBuild = strip.MultiGpu() || ctx->forceStripKernels;
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
    {
        e = LaunchClear(p);
        // the passes of this frame read the staged copy of a guide input (IN_MV is a storage output): it is zeroed too
        const Texture* copy = d->resourcesNum ? &ctx->staged[(uint32_t)d->resources[0].type] : nullptr;
        if (e == cudaSuccess && staged && copy && copy->ptr)
        {
            p.tex[0] = ctx->arena.ToSurf(*copy);
            e = LaunchClear(p);
        }
    }
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
    for (uint32_t i = 0; i < d->resourcesNum && !isClear; i++) // clears zero the ghost rows locally
        if ((pushMask >> i) & 1u)
        {
            const Texture* copy = &ctx->staged[(uint32_t)d->resources[i].type];
            list[n++] = staged && copy->ptr ? copy : Resolve(ctx, d->resources[i].type, d->resources[i].indexInPool); // what the pass wrote
        }
    // (the guide surface needs no push: ClassifyTiles decodes its ghost rows from the ghost rows of the inputs, which arrived with the
    // frame-start push; the barrier below still separates it from the neighbours' far taps, which load the guide from its owner)
    const Result pr = ctx->arena.PushGhostsAndBarrier(list, n, p.stream, ctx->lastError);
    if (timed)
    {
        cudaEventRecord(ctx->timingEvents[3 * slot + 2], p.stream);
        ctx->timingCount = slot + 1;
    }
    return pr == Result::SUCCESS && staged && !isClear ? PullStaged(ctx, d, cs, p.stream) : pr;
}

uint32_t StorageMask(const DispatchDesc* d)
{
    uint32_t m = 0;
    for (uint32_t i = 0; i < d->resourcesNum && i < 32; i++)
        if (d->resources[i].descriptorType == DescriptorType::STORAGE_TEXTURE) m |= 1u << i;
    return m;
}

// frame start: the input strips the application just wrote are pushed to the neighbours' ghost rows, then all ranks meet.
// Frames that stage (StagesInputs, decided from the CommonSettings set last) then gather the guide inputs into their staged
// copies -- own and ghost rows, straight from the inputs through the owner lookup -- and meet once more before any pass reads them.
Result FrameStart(NrdCudaContext* ctx, void* stream)
{
    const Texture* list[std::size(kUserTextures)];
    uint32_t n = 0;
    for (const UserTexture& u : kUserTextures)
        if (u.isInput && ctx->user[(uint32_t)u.type].ptr) list[n++] = &ctx->user[(uint32_t)u.type];
    Result r = ctx->arena.PushGhostsAndBarrier(list, n, (cudaStream_t)stream, ctx->lastError);
    const CommonSettings& cs = ((Scheduler*)ctx->instance)->Common();
    ctx->stagedFrame = false;
    ctx->repartitioned = false;
    if (r != Result::SUCCESS || !StagesInputs(ctx, cs)) return r;
    r = CheckRect(ctx, cs);
    if (r != Result::SUCCESS) return r;
    const int ox = (int)cs.rectOrigin[0], oy = (int)cs.rectOrigin[1], W = ctx->arena.desc.resourceWidth, H = ctx->arena.desc.resourceHeight;
    ShiftedCopyArgs a{};
    a.dx = ox;
    a.dy = oy;
    for (const UserTexture& u : kUserTextures)
    {
        const Texture& copy = ctx->staged[(uint32_t)u.type];
        if (!copy.ptr || !GuideInputRead(u.type, cs) || a.n == kMaxShiftedCopies) continue;
        const Surf dst = ctx->arena.ToSurf(copy); // the rows held locally that lie in the view, i.e. in [0, H - oy)
        a.items[a.n++] = {dst, ctx->arena.ToSurf(ctx->user[(uint32_t)u.type]), 0, W - ox, std::max(dst.ly0, 0), std::min(dst.ly0 + (int)dst.lrows, H - oy),
                          (int)BytesPerTexel(copy.format)};
    }
    cudaEvent_t* ev = TimingSlot(ctx);
    if (ev) cudaEventRecord(ev[0], (cudaStream_t)stream);
    const cudaError_t e = LaunchShiftedCopies(a, false, (cudaStream_t)stream);
    if (ev) cudaEventRecord(ev[1], (cudaStream_t)stream);
    if (e != cudaSuccess) return Fail(ctx, Result::FAILURE, std::string("staged input gather: ") + cudaGetErrorString(e));
    r = ctx->arena.PushGhostsAndBarrier(nullptr, 0, (cudaStream_t)stream, ctx->lastError); // the peers' far taps read these rows
    if (ev) cudaEventRecord(ev[2], (cudaStream_t)stream);
    if (r != Result::SUCCESS) return r;
    ctx->stagedFrame = true;
    ctx->stagedOrigin[0] = (uint32_t)ox;
    ctx->stagedOrigin[1] = (uint32_t)oy;
    return r;
}
} // namespace

extern "C" {

NRD_API Result nrdCudaExecuteDispatch(NrdCudaContext* ctx, const DispatchDesc* d, void* stream)
{
    if (!ctx || !d) return Result::INVALID_ARGUMENT;
    // textures bound in a wider format: convert what this pass reads before it and what it writes after it (nrdCudaDenoise does it per frame)
    Result r = ConvertBound(ctx, d, DescriptorType::TEXTURE, (cudaStream_t)stream);
    if (r == Result::SUCCESS) r = ExecuteInternal(ctx, d, stream, StorageMask(d)); // no look-ahead here: refresh the ghosts of every output
    return r == Result::SUCCESS ? ConvertBound(ctx, d, DescriptorType::STORAGE_TEXTURE, (cudaStream_t)stream) : r;
}

NRD_API Result nrdCudaDenoise(NrdCudaContext* ctx, const Identifier* identifiers, uint32_t identifiersNum, void* stream, uint32_t* launches)
{
    if (!ctx) return Result::INVALID_ARGUMENT;
    const DispatchDesc* dispatches = nullptr;
    uint32_t n = 0;
    Result r = GetComputeDispatches(*ctx->instance, identifiers, identifiersNum, dispatches, n);
    if (r != Result::SUCCESS) return r;
    r = ConvertForeignAll(ctx, true, (cudaStream_t)stream); // inputs bound in a wider format -> the kernels' format
    uint64_t inputs = 0;
    for (const UserTexture& u : kUserTextures)
        if (u.isInput) inputs |= Bit(u.type);
    if (r == Result::SUCCESS) r = ConvertArrays(ctx, inputs, true, (cudaStream_t)stream); // inputs bound as CUDA arrays -> their shadows
    if (r != Result::SUCCESS) return r;
    r = FrameStart(ctx, stream);
    if (r != Result::SUCCESS) return r;
    for (uint32_t i = 0; i < n; i++)
    {
        r = ExecuteInternal(ctx, &dispatches[i], stream, GhostPushMask(dispatches, n, i));
        if (r != Result::SUCCESS) return r;
    }
    r = ConvertForeignAll(ctx, false, (cudaStream_t)stream); // outputs -> the application's wider format
    // every user texture some pass of the frame wrote -> its CUDA array: the outputs, and IN_MV when the frame-0 clear zeroes it or
    // REBLUR TemporalStabilization patches it, so that the array ends the frame as a pointer-bound texture would
    if (r == Result::SUCCESS) r = ConvertArrays(ctx, TypesBoundAs(dispatches, n, DescriptorType::STORAGE_TEXTURE), false, (cudaStream_t)stream);
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

NRD_API Result nrdCudaRepartition(NrdCudaContext* ctx, const uint16_t* stripStarts, void* stream)
{
    if (!ctx) return Result::INVALID_ARGUMENT;
    if (!stripStarts) return Fail(ctx, Result::INVALID_ARGUMENT, "stripStarts is null");
    const std::vector<Texture*> textures = ArenaTextures(ctx);
    const Result r = ctx->arena.Repartition(textures.data(), textures.size(), stripStarts, (cudaStream_t)stream, ctx->lastError);
    if (r == Result::SUCCESS && ctx->arena.strip.MultiGpu())
    {
        // the per-frame state ends with the frame: the next dispatch needs a frame start (input push, staging) under the new table
        ctx->guideValid = false;
        ctx->stagedFrame = false;
        ctx->stagedOrigin[0] = ctx->stagedOrigin[1] = 0;
        ctx->repartitioned = true;
    }
    return r;
}

NRD_API Result nrdCudaSynchronize(NrdCudaContext* ctx, void* stream)
{
    if (!ctx) return Result::INVALID_ARGUMENT;
    cudaError_t e = cudaStreamSynchronize((cudaStream_t)stream);
    if (e != cudaSuccess) return Fail(ctx, Result::FAILURE, std::string("cudaStreamSynchronize: ") + cudaGetErrorString(e));
    return ctx->arena.CheckBarriers(ctx->lastError);
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
