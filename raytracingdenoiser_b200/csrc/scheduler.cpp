// Pass scheduler core -- see scheduler.h.  No GPU calls.
#include "scheduler.h"

#include <algorithm>
#include <cassert>
#include <cstdio>
#include <cstring>

using namespace nrd;

namespace nrdb200
{
static bool IsIntegerFormat(Format f)
{
#define NRD_B200_ISINT(name, bytes, isInt) isInt != 0,
    static const bool table[] = {NRD_B200_FORMATS(NRD_B200_ISINT)};
#undef NRD_B200_ISINT
    return table[(size_t)f];
}

static const Sampler kSamplers[] = {Sampler::NEAREST_CLAMP, Sampler::LINEAR_CLAMP};

static inline uint16_t CeilDiv(uint32_t x, uint16_t y) { return uint16_t((x + y - 1) / y); }

static bool Contains(Identifier id, const Identifier* ids, uint32_t n)
{
    for (uint32_t i = 0; i < n; i++)
        if (ids[i] == id) return true;
    return false;
}

Scheduler::Scheduler(const MemoryHooks& hooks)
    : hooks_(hooks), slots_(HookAllocator<DenoiserSlot>(&hooks_)), permanentPool_(HookAllocator<TextureDesc>(&hooks_)),
      transientPool_(HookAllocator<TextureDesc>(&hooks_)), resources_(HookAllocator<ResourceDesc>(&hooks_)),
      clears_(HookAllocator<ClearTarget>(&hooks_)), pingPongs_(HookAllocator<PingPong>(&hooks_)),
      ranges_(HookAllocator<ResourceRangeDesc>(&hooks_)), pipelineRangeOffset_(HookAllocator<size_t>(&hooks_)),
      pipelines_(HookAllocator<PipelineDesc>(&hooks_)), pipelineKinds_(HookAllocator<PassKind>(&hooks_)),
      passes_(HookAllocator<PassTemplate>(&hooks_)), active_(HookAllocator<DispatchDesc>(&hooks_)),
      transientRemap_(HookAllocator<uint16_t>(&hooks_)), ownedStrings_(HookAllocator<char*>(&hooks_))
{
    constantArenaRaw_ = (uint8_t*)hooks_.alloc(kConstantArenaSize + 16, 16);
    constantArena_ = (uint8_t*)(((uintptr_t)constantArenaRaw_ + 15) & ~(uintptr_t)15);
    memset(constantArena_, 0, kConstantArenaSize);
}

Scheduler::~Scheduler()
{
    for (char* s : ownedStrings_) hooks_.free(s);
    hooks_.free(constantArenaRaw_);
}

// ---------------------------------------------------------------------------------------------
// Creation (reference: InstanceImpl.cpp:100-267)
// ---------------------------------------------------------------------------------------------
Result Scheduler::Create(const InstanceCreationDesc& creation)
{
    const LibraryDesc& lib = GetLibraryDesc();

    for (uint32_t i = 0; i < creation.denoisersNum; i++)
    {
        const DenoiserDesc& dd = creation.denoisers[i];

        bool supported = false;
        for (uint32_t j = 0; j < lib.supportedDenoisersNum; j++)
            supported |= lib.supportedDenoisers[j] == dd.denoiser;
        if (!supported) return Result::UNSUPPORTED;

        for (uint32_t j = 0; j < creation.denoisersNum; j++)
            if (j != i && creation.denoisers[j].identifier == dd.identifier) return Result::NON_UNIQUE_IDENTIFIER;

        permanentOffset_ = (uint16_t)permanentPool_.size();
        transientOffset_ = (uint16_t)transientPool_.size();
        transientRemap_.clear();

        DenoiserSlot slot;
        memset((void*)&slot, 0, sizeof(slot));
        slot.desc = dd;
        slot.firstPass = passes_.size();
        slot.firstPingPong = pingPongs_.size();
        const size_t firstResource = resources_.size();

        switch (dd.denoiser)
        {
            case Denoiser::REBLUR_DIFFUSE: AddReblur(slot, true, false); break;
            case Denoiser::REBLUR_SPECULAR: AddReblur(slot, false, true); break;
            case Denoiser::REBLUR_DIFFUSE_SPECULAR: AddReblur(slot, true, true); break;
            case Denoiser::RELAX_DIFFUSE: AddRelax(slot, true, false); break;
            case Denoiser::RELAX_SPECULAR: AddRelax(slot, false, true); break;
            case Denoiser::RELAX_DIFFUSE_SPECULAR: AddRelax(slot, true, true); break;
            case Denoiser::SIGMA_SHADOW: AddSigmaShadow(slot, false); break;
            case Denoiser::SIGMA_SHADOW_TRANSLUCENCY: AddSigmaShadow(slot, true); break;
            case Denoiser::REFERENCE: AddReference(slot); break;
            default: return Result::INVALID_ARGUMENT;
        }

        slot.pingPongNum = pingPongs_.size() - slot.firstPingPong;
        for (size_t p = slot.firstPass; p < passes_.size(); p++) passes_[p].identifier = dd.identifier;

        // every texture bound as storage anywhere (plus its ping-pong partner) must be cleared on CLEAR_AND_RESTART
        for (size_t r = firstResource; r < resources_.size(); r++)
        {
            const ResourceDesc& res = resources_[r];
            if (res.descriptorType != DescriptorType::STORAGE_TEXTURE || res.type == ResourceType::OUT_VALIDATION) continue;

            bool known = false;
            for (const ClearTarget& c : clears_)
                known |= c.resource.descriptorType == res.descriptorType && c.resource.type == res.type && c.resource.indexInPool == res.indexInPool;
            if (known) continue;

            bool isInteger = false;
            uint16_t downsample = 1;
            if (res.type == ResourceType::PERMANENT_POOL || res.type == ResourceType::TRANSIENT_POOL)
            {
                const TextureDesc& td = res.type == ResourceType::PERMANENT_POOL ? permanentPool_[res.indexInPool] : transientPool_[res.indexInPool];
                isInteger = IsIntegerFormat(td.format);
                downsample = td.downsampleFactor;
            }
            clears_.push_back({dd.identifier, res, downsample, isInteger});

            for (size_t p = 0; p < slot.pingPongNum; p++)
            {
                const PingPong& pp = pingPongs_[slot.firstPingPong + p];
                if (pp.resourceIndex == r)
                {
                    clears_.push_back({dd.identifier, {res.descriptorType, res.type, pp.other}, downsample, isInteger});
                    break;
                }
            }
        }
        slots_.push_back(slot);
    }

    // two generic clear pipelines (float / uint)
    clearPass_[0] = passes_.size();
    passName_ = "Clear (f)";
    passResourceOffset_ = resources_.size();
    Out(0);
    Emit({Family::CLEAR, Pass::Float}, 16, 16, 0);

    clearPass_[1] = passes_.size();
    passName_ = "Clear (ui)";
    passResourceOffset_ = resources_.size();
    Out(0);
    Emit({Family::CLEAR, Pass::Uint}, 16, 16, 0);

    FinalizeDesc();
    return Result::SUCCESS;
}

void Scheduler::AddTransient(Format f, uint16_t downsample)
{
    // reuse a transient texture of an earlier denoiser of this instance when format and size match and it is not yet
    // taken by the current denoiser (reference: InstanceImpl.cpp:773-803)
    for (uint16_t i = 0; i < transientOffset_; i++)
    {
        const TextureDesc& t = transientPool_[i];
        if (t.format != f || t.downsampleFactor != downsample) continue;
        if (std::find(transientRemap_.begin(), transientRemap_.end(), i) == transientRemap_.end())
        {
            transientRemap_.push_back(i);
            return;
        }
    }
    transientRemap_.push_back((uint16_t)transientPool_.size());
    transientPool_.push_back({f, downsample});
}

void Scheduler::BeginPass(const char* denoiserName, const char* passName)
{
    size_t n = strlen(denoiserName) + 3 + strlen(passName) + 1;
    char* s = (char*)hooks_.alloc(n, 1);
    snprintf(s, n, "%s - %s", denoiserName, passName);
    ownedStrings_.push_back(s);
    passName_ = s;
    passResourceOffset_ = resources_.size();
}

void Scheduler::PushResource(DescriptorType type, uint16_t localId, uint16_t swapWith)
{
    ResourceType resourceType = (ResourceType)localId;
    uint16_t index = 0;
    if (localId >= kTransientBase)
    {
        resourceType = ResourceType::TRANSIENT_POOL;
        index = transientRemap_[localId - kTransientBase];
        if (swapWith != kNoSwap) pingPongs_.push_back({resources_.size(), transientRemap_[swapWith - kTransientBase]});
    }
    else if (localId >= kPermanentBase)
    {
        resourceType = ResourceType::PERMANENT_POOL;
        index = uint16_t(permanentOffset_ + localId - kPermanentBase);
        if (swapWith != kNoSwap) pingPongs_.push_back({resources_.size(), uint16_t(permanentOffset_ + swapWith - kPermanentBase)});
    }
    resources_.push_back({type, resourceType, index});
}

// "<family>[_Perf][_<signals>]_<pass>.cs", e.g. REBLUR_Perf_DiffuseSpecular_Blur.cs, SIGMA_ShadowTranslucency_Blur.cs, Clear_Float.cs
static void ShaderFileName(const PassKind& k, char* out, size_t size)
{
    static const char* const kFamilies[] = {"Clear", "REBLUR", "RELAX", "SIGMA", "REFERENCE"};
#define NRD_B200_PASS_NAME(name) #name,
    static const char* const kPasses[] = {NRD_B200_PASSES(NRD_B200_PASS_NAME)};
#undef NRD_B200_PASS_NAME
    static const char* const kSignals[] = {"", "Diffuse", "Specular", "DiffuseSpecular", "Shadow"};
    const char* signal = k.translucent ? "ShadowTranslucency" : kSignals[k.signals];
    snprintf(out, size, "%s%s%s%s_%s.cs", kFamilies[(int)k.family], k.perf ? "_Perf" : "", *signal ? "_" : "", signal, kPasses[(int)k.pass]);
}

void Scheduler::Emit(const PassKind& kind, uint8_t threadsX, uint8_t threadsY, uint32_t constantSize, uint16_t downsample, uint16_t maxRepeats)
{
    // pipelines are unique per shader file name (reference: InstanceImpl.cpp:592-633)
    char shaderFileName[80];
    ShaderFileName(kind, shaderFileName, sizeof(shaderFileName));
    size_t pipelineIndex = 0;
    for (; pipelineIndex < pipelines_.size(); pipelineIndex++)
        if (!strcmp(pipelines_[pipelineIndex].shaderFileName, shaderFileName)) break;

    if (pipelineIndex == pipelines_.size())
    {
        const size_t n = strlen(shaderFileName) + 1;
        char* name = (char*)hooks_.alloc(n, 1);
        memcpy(name, shaderFileName, n);
        ownedStrings_.push_back(name);
        pipelineKinds_.push_back(kind);
        PipelineDesc pd{};
        pd.shaderFileName = name;
        pd.shaderEntryPointName = "main";
        pd.hasConstantData = constantSize != 0;
        pipelineRangeOffset_.push_back(ranges_.size());
        for (int r = 0; r < 2; r++)
        {
            ResourceRangeDesc range{};
            range.descriptorType = r == 0 ? DescriptorType::TEXTURE : DescriptorType::STORAGE_TEXTURE;
            for (size_t i = passResourceOffset_; i < resources_.size(); i++)
                if (resources_[i].descriptorType == range.descriptorType) range.descriptorsNum++;
            if (range.descriptorsNum)
            {
                ranges_.push_back(range);
                pd.resourceRangesNum++;
            }
        }
        pipelines_.push_back(pd);
    }

    PassTemplate pt{};
    pt.name = passName_;
    pt.resourceOffset = passResourceOffset_;
    pt.resourcesNum = uint32_t(resources_.size() - passResourceOffset_);
    pt.constantSize = constantSize;
    pt.pipelineIndex = (uint16_t)pipelineIndex;
    pt.downsample = downsample;
    pt.maxRepeats = maxRepeats;
    pt.threadsX = threadsX;
    pt.threadsY = threadsY;
    passes_.push_back(pt);
}

void Scheduler::FinalizeDesc()
{
    desc_ = {};
    desc_.constantBufferRegisterIndex = 0;
    desc_.constantBufferSpaceIndex = 0;
    desc_.samplers = kSamplers;
    desc_.samplersNum = 2;
    desc_.samplersSpaceIndex = 0;
    desc_.samplersBaseRegisterIndex = 0;
    desc_.resourcesSpaceIndex = 0;

    for (size_t i = 0; i < pipelines_.size(); i++) pipelines_[i].resourceRanges = ranges_.data() + pipelineRangeOffset_[i];
    desc_.pipelines = pipelines_.data();
    desc_.pipelinesNum = (uint32_t)pipelines_.size();
    desc_.permanentPool = permanentPool_.data();
    desc_.permanentPoolSize = (uint32_t)permanentPool_.size();
    desc_.transientPool = transientPool_.data();
    desc_.transientPoolSize = (uint32_t)transientPool_.size();

    // descriptor budget, as an RHI-based caller would need it (reference: InstanceImpl.cpp:671-724; all spaces are 0,
    // so samplers live in the same set as everything else and there is a single descriptor set per dispatch)
    DescriptorPoolDesc& dp = desc_.descriptorPoolDesc;
    for (const PassTemplate& p : passes_)
    {
        for (uint32_t i = 0; i < p.resourcesNum; i++)
        {
            if (resources_[p.resourceOffset + i].descriptorType == DescriptorType::TEXTURE)
                dp.texturesMaxNum += p.maxRepeats;
            else
                dp.storageTexturesMaxNum += p.maxRepeats;
        }
        dp.setsMaxNum += p.maxRepeats;
        dp.samplersMaxNum += p.maxRepeats * desc_.samplersNum;
        if (p.constantSize)
        {
            dp.constantBuffersMaxNum += p.maxRepeats;
            desc_.constantBufferMaxDataSize = std::max(desc_.constantBufferMaxDataSize, p.constantSize);
        }
    }
    uint32_t clearNum = (uint32_t)clears_.size();
    dp.storageTexturesMaxNum += clearNum;
    dp.setsMaxNum += clearNum;
    dp.samplersMaxNum += clearNum * desc_.samplersNum;
}

// ---------------------------------------------------------------------------------------------
// Per frame (reference: InstanceImpl.cpp:269-473)
// ---------------------------------------------------------------------------------------------
Result Scheduler::SetCommonSettings(const CommonSettings& s)
{
    splitScreenPrev = common_.splitScreen;
    common_ = s;

    if (firstUse_)
    {
        common_.accumulationMode = AccumulationMode::CLEAR_AND_RESTART;
        firstUse_ = false;
    }

    if (common_.accumulationMode != AccumulationMode::CONTINUE)
    {
        // history is discarded: "previous" state collapses onto the state of the last call
        // (the reference also copies its current matrices into the "prev" members here, InstanceImpl.cpp:286-287, but then
        // unconditionally reloads them from the settings, :360-382 -- so after a reset the application's *Prev matrices
        // are still the ones used; same here)
        splitScreenPrev = 0.0f;
        for (int i = 0; i < 2; i++)
        {
            common_.resourceSizePrev[i] = common_.resourceSize[i];
            common_.rectSizePrev[i] = common_.rectSize[i];
            common_.cameraJitterPrev[i] = common_.cameraJitter[i];
        }
    }

    bool ok = common_.viewZScale > 0.0f;
    ok &= common_.resourceSize[0] != 0 && common_.resourceSize[1] != 0;
    ok &= common_.resourceSizePrev[0] != 0 && common_.resourceSizePrev[1] != 0;
    ok &= common_.rectSize[0] != 0 && common_.rectSize[1] != 0;
    ok &= common_.rectSizePrev[0] != 0 && common_.rectSizePrev[1] != 0;
    ok &= (common_.motionVectorScale[0] != 0.0f && common_.motionVectorScale[1] != 0.0f) || common_.isMotionVectorInWorldSpace;
    for (int i = 0; i < 2; i++)
    {
        ok &= common_.cameraJitter[i] >= -0.5f && common_.cameraJitter[i] <= 0.5f;
        ok &= common_.cameraJitterPrev[i] >= -0.5f && common_.cameraJitterPrev[i] <= 0.5f;
    }
    ok &= common_.denoisingRange > 0.0f;
    ok &= common_.disocclusionThreshold > 0.0f;
    ok &= common_.disocclusionThresholdAlternate > 0.0f;
    // strandMaterialID / cameraAttachedReflectionMaterialID == 0 would need the material bits: this build always has them
    // (NormalEncoding::R10_G10_B10_A2_UNORM), so those two reference checks always pass.

    // blur kernel rotators, one per frame (reference: InstanceImpl.cpp:339-349)
    const uint32_t fi = common_.frameIndex;
    rotatorPre = GetRotator(Weyl1D(0.5f, fi) * Radians(90.0f));
    rotator = CombineRotators(GetRotator(Weyl1D(0.0f, fi * 2) * Radians(90.0f)), GetRotator(Bayer4x4(0, 0, fi * 2) * Radians(360.0f)));
    rotatorPost = CombineRotators(GetRotator(Weyl1D(0.0f, fi * 2 + 1) * Radians(90.0f)), GetRotator(Bayer4x4(0, 0, fi * 2 + 1) * Radians(360.0f)));

    viewToClip = Mat4::FromColumnMajor(common_.viewToClipMatrix);
    viewToClipPrev = Mat4::FromColumnMajor(common_.viewToClipMatrixPrev);
    worldToView = Mat4::FromColumnMajor(common_.worldToViewMatrix);
    worldToViewPrev = Mat4::FromColumnMajor(common_.worldToViewMatrixPrev);
    worldPrevToWorld = Mat4::FromColumnMajor(common_.worldPrevToWorldMatrix);
    uint32_t flags = 0;
    float project[3];
    DecomposeProjection(viewToClip, flags, frustum, project);
    if (!(flags & PROJ_LEFT_HANDED))
    {
        // right-handed input: flip view-space z everywhere so the kernels only ever see left-handed matrices
        viewToClip.negateColumn(2);
        viewToClipPrev.negateColumn(2);
        worldToView.negateRow(2);
        worldToViewPrev.negateRow(2);
    }

    viewToWorld = worldToView;
    viewToWorld.invertOrtho();
    viewToWorldPrev = worldToViewPrev;
    viewToWorldPrev.invertOrtho();

    const Vec3 camPos = viewToWorld.translation();
    const Vec3 camPosPrev = viewToWorldPrev.translation();
    const Vec3 delta = {camPosPrev.x - camPos.x, camPosPrev.y - camPos.y, camPosPrev.z - camPos.z};

    // camera-relative matrices: the current camera sits at the origin, the previous one at `delta`
    viewToWorld.setTranslation({0.0f, 0.0f, 0.0f});
    worldToView = viewToWorld;
    worldToView.invertOrtho();
    viewToWorldPrev.setTranslation(delta);
    worldToViewPrev = viewToWorldPrev;
    worldToViewPrev.invertOrtho();

    worldToClip = viewToClip * worldToView;
    worldToClipPrev = viewToClipPrev * worldToViewPrev;

    DecomposeProjection(viewToClip, flags, frustum, project);
    projectY = project[1];
    orthoMode = (flags & PROJ_ORTHO) ? -1.0f : 0.0f;
    uint32_t flagsPrev = 0;
    DecomposeProjection(viewToClipPrev, flagsPrev, frustumPrev, nullptr);

    viewDirection = {-viewToWorld.at(0, 2), -viewToWorld.at(1, 2), -viewToWorld.at(2, 2)};
    viewDirectionPrev = {-viewToWorldPrev.at(0, 2), -viewToWorldPrev.at(1, 2), -viewToWorldPrev.at(2, 2)};
    cameraDelta = delta;

    // frame time: user provided, else smoothed wall clock (reference: Source/Timer.cpp:58-66)
    auto now = std::chrono::steady_clock::now();
    if (hasPrevTime_)
    {
        float ms = std::chrono::duration<float, std::milli>(now - prevTime_).count();
        float rel = std::fabs(ms - smoothedTimeDelta_) / (std::min(ms, smoothedTimeDelta_) + 1e-7f);
        float f = rel / (1.0f + rel);
        smoothedTimeDelta_ += (ms - smoothedTimeDelta_) * std::max(f, 1.0f / 32.0f);
    }
    prevTime_ = now;
    hasPrevTime_ = true;

    timeDelta = common_.timeDeltaBetweenFrames > 0.0f ? common_.timeDeltaBetweenFrames : smoothedTimeDelta_;
    frameRateScale = std::max(33.333f / timeDelta, 1.0f);

    float dx = std::fabs(common_.cameraJitter[0] - common_.cameraJitterPrev[0]);
    float dy = std::fabs(common_.cameraJitter[1] - common_.cameraJitterPrev[1]);
    jitterDelta = std::max(dx, dy);

    float fps = frameRateScale * 30.0f;
    float nonLinearAccumSpeed = fps * 0.25f / (1.0f + fps * 0.25f);
    checkerboardResolveAccumSpeed = nonLinearAccumSpeed + (0.5f - nonLinearAccumSpeed) * jitterDelta;

    return ok ? Result::SUCCESS : Result::INVALID_ARGUMENT;
}

Result Scheduler::SetDenoiserSettings(Identifier id, const void* settings)
{
    for (DenoiserSlot& slot : slots_)
        if (slot.desc.identifier == id)
        {
            memcpy(&slot.settings, settings, slot.settingsSize);
            return Result::SUCCESS;
        }
    return Result::INVALID_ARGUMENT;
}

void Scheduler::SwapPingPongs(const DenoiserSlot& slot)
{
    for (size_t i = 0; i < slot.pingPongNum; i++)
    {
        PingPong& pp = pingPongs_[slot.firstPingPong + i];
        std::swap(resources_[pp.resourceIndex].indexInPool, pp.other);
    }
}

Result Scheduler::GetComputeDispatches(const Identifier* ids, uint32_t idsNum, const DispatchDesc*& out, uint32_t& outNum)
{
    constantOffset_ = 0;
    active_.clear();

    if (!ids || !idsNum)
    {
        out = nullptr;
        outNum = 0;
        return !idsNum ? Result::SUCCESS : Result::INVALID_ARGUMENT;
    }

    if (common_.accumulationMode == AccumulationMode::CLEAR_AND_RESTART)
    {
        for (const ClearTarget& c : clears_)
        {
            if (!Contains(c.identifier, ids, idsNum)) continue;
            const PassTemplate& pt = passes_[clearPass_[c.isInteger ? 1 : 0]];
            uint16_t w = CeilDiv(common_.resourceSize[0], c.downsample);
            uint16_t h = CeilDiv(common_.resourceSize[1], c.downsample);
            DispatchDesc d{};
            d.name = pt.name;
            d.identifier = c.identifier;
            d.resources = &c.resource;
            d.resourcesNum = 1;
            d.pipelineIndex = pt.pipelineIndex;
            d.gridWidth = CeilDiv(w, pt.threadsX);
            d.gridHeight = CeilDiv(h, pt.threadsY);
            active_.push_back(d);
        }
    }

    for (const DenoiserSlot& slot : slots_)
    {
        if (!Contains(slot.desc.identifier, ids, idsNum)) continue;
        SwapPingPongs(slot);
        switch (slot.desc.denoiser)
        {
            case Denoiser::REBLUR_DIFFUSE:
            case Denoiser::REBLUR_SPECULAR:
            case Denoiser::REBLUR_DIFFUSE_SPECULAR: UpdateReblur(slot); break;
            case Denoiser::RELAX_DIFFUSE:
            case Denoiser::RELAX_SPECULAR:
            case Denoiser::RELAX_DIFFUSE_SPECULAR: UpdateRelax(slot); break;
            case Denoiser::SIGMA_SHADOW:
            case Denoiser::SIGMA_SHADOW_TRANSLUCENCY: UpdateSigma(slot); break;
            case Denoiser::REFERENCE: UpdateReference(slot); break;
            default: break;
        }
    }

    // tell the executor when a constant block is byte-identical to the previous one (no re-upload needed)
    for (size_t i = 1; i < active_.size(); i++)
    {
        const DispatchDesc& prev = active_[i - 1];
        DispatchDesc& cur = active_[i];
        if (prev.constantBufferDataSize == cur.constantBufferDataSize &&
            !memcmp(prev.constantBufferData, cur.constantBufferData, cur.constantBufferDataSize))
            cur.constantBufferDataMatchesPreviousDispatch = true;
    }

    out = active_.data();
    outNum = (uint32_t)active_.size();
    return outNum ? Result::SUCCESS : Result::INVALID_ARGUMENT;
}

void* Scheduler::Push(const DenoiserSlot& slot, uint32_t localPassIndex)
{
    const PassTemplate& pt = passes_[slot.firstPass + localPassIndex];

    DispatchDesc d{};
    d.name = pt.name;
    d.identifier = pt.identifier;
    d.resources = resources_.data() + pt.resourceOffset;
    d.resourcesNum = pt.resourcesNum;
    d.pipelineIndex = pt.pipelineIndex;
    d.constantBufferDataSize = pt.constantSize;
    // blocks are placed on 16-byte boundaries and zero-padded to whole registers: the reported size is the reference's
    // sizeof(), the kernels copy whole register-aligned structs (csrc/constants.h)
    const uint32_t paddedSize = (pt.constantSize + 15u) & ~15u;
    if (constantOffset_ + paddedSize <= kConstantArenaSize)
    {
        d.constantBufferData = constantArena_ + constantOffset_;
        memset((void*)d.constantBufferData, 0, paddedSize);
    }
    constantOffset_ += paddedSize;

    uint16_t w = common_.rectSize[0], h = common_.rectSize[1], ds = pt.downsample;
    if (ds == kUseMaxDims)
    {
        w = std::max(w, common_.rectSizePrev[0]);
        h = std::max(h, common_.rectSizePrev[1]);
        ds = 1;
    }
    else if (ds == kIgnoreRect)
    {
        w = common_.resourceSize[0];
        h = common_.resourceSize[1];
        ds = 1;
    }
    w = CeilDiv(w, ds);
    h = CeilDiv(h, ds);
    d.gridWidth = CeilDiv(w, pt.threadsX);
    d.gridHeight = CeilDiv(h, pt.threadsY);

    active_.push_back(d);
    return (void*)d.constantBufferData;
}
} // namespace nrdb200
