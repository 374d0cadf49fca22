// Pass scheduler: turns CommonSettings + per-denoiser settings into the per-frame DispatchDesc[] stream.
// Behavioural restatement of the reference's Source/InstanceImpl.{h,cpp} (Create :100-267, SetCommonSettings :269-473,
// GetComputeDispatches :490-578, pipeline dedup :580-647, PrepareDesc :649-725, ping-pong :727-736, transient pool
// aliasing :773-803, grid sizing :805-862) with its own data structures.  It makes no GPU calls.
#pragma once
#include "../../include/nrd_b200.h"
#include "constants.h"
#include "hostmath.h"
#include "passes.h"

#include <chrono>
#include <new>
#include <vector>

namespace nrdb200
{
using namespace nrdb200_abi; // PassKind (passes.h)

// STL allocator over the user's AllocationCallbacks (reference: Source/StdAllocator.h)
struct MemoryHooks
{
    nrd::AllocationCallbacks cb;
    void* alloc(size_t size, size_t align) const { return cb.Allocate(cb.userArg, size, align); }
    void free(void* p) const { cb.Free(cb.userArg, p); }
};

template <class T> struct HookAllocator
{
    typedef T value_type;
    const MemoryHooks* hooks;
    explicit HookAllocator(const MemoryHooks* h) : hooks(h) {}
    template <class U> HookAllocator(const HookAllocator<U>& o) : hooks(o.hooks) {}
    T* allocate(size_t n) { return (T*)hooks->alloc(n * sizeof(T), alignof(T) < 16 ? 16 : alignof(T)); }
    void deallocate(T* p, size_t) { hooks->free(p); }
    template <class U> bool operator==(const HookAllocator<U>& o) const { return hooks == o.hooks; }
    template <class U> bool operator!=(const HookAllocator<U>& o) const { return hooks != o.hooks; }
};
template <class T> using Vec = std::vector<T, HookAllocator<T>>;

constexpr uint16_t kPermanentBase = 1000; // local resource ids >= this address the permanent pool
constexpr uint16_t kTransientBase = 2000; // ... and >= this the transient pool
constexpr uint16_t kNoSwap = 0xFFFF;
constexpr uint16_t kUseMaxDims = 0xFFFF;  // grid from max(rect, rectPrev)
constexpr uint16_t kIgnoreRect = 0xFFFE;  // grid from resourceSize
constexpr size_t kConstantArenaSize = 128 * 1024;

union AnySettings
{
    nrd::ReblurSettings reblur;
    nrd::RelaxSettings relax;
    nrd::SigmaSettings sigma;
    nrd::ReferenceSettings reference;
    AnySettings() {}
};

struct DenoiserSlot
{
    nrd::DenoiserDesc desc;
    AnySettings settings;
    size_t settingsSize;
    size_t firstPass;     // index of this denoiser's pass 0 in passes_
    size_t firstPingPong; // range in pingPongs_
    size_t pingPongNum;
};

struct PingPong
{
    size_t resourceIndex; // into resources_
    uint16_t other;       // pool index to swap with
};

struct PassTemplate
{
    const char* name;
    size_t resourceOffset;
    uint32_t resourcesNum;
    uint32_t constantSize;
    nrd::Identifier identifier;
    uint16_t pipelineIndex;
    uint16_t downsample;
    uint16_t maxRepeats;
    uint8_t threadsX, threadsY;
};

struct ClearTarget
{
    nrd::Identifier identifier;
    nrd::ResourceDesc resource;
    uint16_t downsample;
    bool isInteger;
};

class Scheduler
{
public:
    explicit Scheduler(const MemoryHooks& hooks);
    ~Scheduler();

    nrd::Result Create(const nrd::InstanceCreationDesc& desc);
    nrd::Result SetCommonSettings(const nrd::CommonSettings& s);
    nrd::Result SetDenoiserSettings(nrd::Identifier id, const void* settings);
    nrd::Result GetComputeDispatches(const nrd::Identifier* ids, uint32_t idsNum, const nrd::DispatchDesc*& out, uint32_t& outNum);
    const nrd::InstanceDesc& GetDesc() const { return desc_; }
    const MemoryHooks& Hooks() const { return hooks_; }
    const nrd::CommonSettings& Common() const { return common_; }
    const PassKind& PipelineKind(size_t pipelineIndex) const { return pipelineKinds_[pipelineIndex]; }
    bool HasDenoiser(nrd::Denoiser d) const
    {
        for (size_t i = 0; i < slots_.size(); i++)
            if (slots_[i].desc.denoiser == d) return true;
        return false;
    }

    // ---- recipe building blocks (used by recipes_*.cpp) ----
    void AddPermanent(nrd::Format f, uint16_t downsample = 1) { permanentPool_.push_back({f, downsample}); }
    void AddTransient(nrd::Format f, uint16_t downsample = 1);
    void BeginPass(const char* denoiserName, const char* passName);
    void In(uint16_t localId, uint16_t swapWith = kNoSwap) { PushResource(nrd::DescriptorType::TEXTURE, localId, swapWith); }
    void Out(uint16_t localId, uint16_t swapWith = kNoSwap) { PushResource(nrd::DescriptorType::STORAGE_TEXTURE, localId, swapWith); }
    void Emit(const PassKind& kind, uint8_t threadsX, uint8_t threadsY, uint32_t constantSize, uint16_t downsample = 1, uint16_t maxRepeats = 1);
    void* Push(const DenoiserSlot& slot, uint32_t localPassIndex); // activates a pass for this frame, returns its constant block

    // ---- per-frame derived camera state (read by the recipes when they fill constants) ----
    Mat4 viewToClip = Mat4::Identity(), viewToClipPrev = Mat4::Identity();
    Mat4 worldToView = Mat4::Identity(), worldToViewPrev = Mat4::Identity();
    Mat4 viewToWorld = Mat4::Identity(), viewToWorldPrev = Mat4::Identity();
    Mat4 worldToClip = Mat4::Identity(), worldToClipPrev = Mat4::Identity();
    Mat4 worldPrevToWorld = Mat4::Identity();
    Vec4 rotatorPre{}, rotator{}, rotatorPost{};
    float frustum[4] = {}, frustumPrev[4] = {};
    Vec3 cameraDelta{}, viewDirection{}, viewDirectionPrev{};
    float splitScreenPrev = 0.0f, orthoMode = 0.0f, checkerboardResolveAccumSpeed = 0.0f, jitterDelta = 0.0f;
    float timeDelta = 0.0f, frameRateScale = 0.0f, projectY = 0.0f;

private:
    void PushResource(nrd::DescriptorType type, uint16_t localId, uint16_t swapWith);
    void FinalizeDesc();
    void SwapPingPongs(const DenoiserSlot& slot);

    // recipes (recipes_reblur.cpp / recipes_relax.cpp / recipes_sigma.cpp)
    void AddReblur(DenoiserSlot& slot, bool hasDiffuse, bool hasSpecular);
    void UpdateReblur(const DenoiserSlot& slot);
    void FillReblurConstants(const nrd::ReblurSettings& s, void* data);
    void AddRelax(DenoiserSlot& slot, bool hasDiff, bool hasSpec);
    void UpdateRelax(const DenoiserSlot& slot);
    void FillRelaxConstants(const nrd::RelaxSettings& s, void* data);
    void AddSigmaShadow(DenoiserSlot& slot, bool translucent);
    void UpdateSigma(const DenoiserSlot& slot);
    void FillSigmaConstants(const nrd::SigmaSettings& s, void* data);
    void AddReference(DenoiserSlot& slot);
    void UpdateReference(const DenoiserSlot& slot);

    MemoryHooks hooks_;
    Vec<DenoiserSlot> slots_;
    Vec<nrd::TextureDesc> permanentPool_, transientPool_;
    Vec<nrd::ResourceDesc> resources_;
    Vec<ClearTarget> clears_;
    Vec<PingPong> pingPongs_;
    Vec<nrd::ResourceRangeDesc> ranges_;
    Vec<size_t> pipelineRangeOffset_;
    Vec<nrd::PipelineDesc> pipelines_;
    Vec<PassKind> pipelineKinds_; // one per pipeline
    Vec<PassTemplate> passes_;
    Vec<nrd::DispatchDesc> active_;
    Vec<uint16_t> transientRemap_;
    Vec<char*> ownedStrings_;
    nrd::InstanceDesc desc_{};
    nrd::CommonSettings common_{};
    uint8_t* constantArenaRaw_ = nullptr;
    uint8_t* constantArena_ = nullptr;
    size_t constantOffset_ = 0;
    size_t passResourceOffset_ = 0;
    const char* passName_ = nullptr;
    size_t clearPass_[2] = {};
    uint16_t permanentOffset_ = 0, transientOffset_ = 0;
    bool firstUse_ = true;
    bool hasPrevTime_ = false;
    std::chrono::steady_clock::time_point prevTime_;
    float smoothedTimeDelta_ = 16.6667f;
    uint32_t accumulatedFrameNum_ = 0; // REFERENCE denoiser: frames accumulated so far (one counter per instance, like the reference)
};
} // namespace nrdb200
