// RELAX_DIFFUSE_SPECULAR pass graph and per-frame schedule.
// Restates the reference's Source/Denoisers/Relax_DiffuseSpecular.hpp (pools, bindings, A-trous binding variants) and
// Source/Relax.cpp:60-180 (AddSharedConstants_Relax), :182-295 (Update_Relax).
#include "scheduler.h"

#include <algorithm>
#include <cmath>
#include <cstring>

using namespace nrd;

namespace nrdb200
{
namespace
{
constexpr uint16_t R(ResourceType t) { return (uint16_t)t; }
constexpr uint16_t kDummy = R(ResourceType::IN_VIEWZ);
constexpr uint32_t kMaxAtrousPasses = 8;
constexpr uint32_t kAtrousBindingVariants = 5;

enum RelaxPass : uint32_t
{
    RX_CLASSIFY_TILES = 0,
    RX_HITDIST_RECONSTRUCTION = 1,                          // 2
    RX_PREPASS = RX_HITDIST_RECONSTRUCTION + 2,             // 2
    RX_TEMPORAL_ACCUMULATION = RX_PREPASS + 2,              // 4
    RX_HISTORY_FIX = RX_TEMPORAL_ACCUMULATION + 4,
    RX_HISTORY_CLAMPING,
    RX_COPY,
    RX_ANTI_FIREFLY,
    RX_ATROUS,                                              // 2 x 5 binding variants
    RX_SPLIT_SCREEN = RX_ATROUS + 2 * kAtrousBindingVariants,
    RX_VALIDATION,
};

const uint32_t kSharedSize = offsetof(RelaxConstants, gStepSize); // 704
} // namespace

// One builder for Source/Denoisers/Relax_Diffuse.hpp, Relax_Specular.hpp and Relax_DiffuseSpecular.hpp: the one-signal graphs are
// the two-signal graph without the other signal's textures and bindings (pool order: Relax_Diffuse.hpp:17-44, Relax_Specular.hpp:17-52,
// Relax_DiffuseSpecular.hpp:17-62).
void Scheduler::AddRelax(DenoiserSlot& slot, bool hasDiff, bool hasSpec)
{
    new (&slot.settings.relax) RelaxSettings();
    slot.settingsSize = sizeof(RelaxSettings);
    const uint8_t signals = (hasDiff ? SIGNAL_DIFFUSE : 0) | (hasSpec ? SIGNAL_SPECULAR : 0);
    const char* dn = hasDiff && hasSpec ? "RELAX_DiffuseSpecular" : (hasSpec ? "RELAX_Specular" : "RELAX_Diffuse");
    const uint32_t cb = kSharedSize;
    const uint32_t cbAtrous = offsetof(RelaxConstants, gIsLastPass) + sizeof(uint32_t); // 712: sizeof() of the reference struct, no register padding

    uint16_t next = kPermanentBase;
    uint16_t P_SPEC_ILLUM_PREV = 0, P_DIFF_ILLUM_PREV = 0, P_SPEC_ILLUM_RESPONSIVE_PREV = 0, P_DIFF_ILLUM_RESPONSIVE_PREV = 0, P_REFLECTION_HIT_T_CURR = 0, P_REFLECTION_HIT_T_PREV = 0;
    if (hasSpec) { P_SPEC_ILLUM_PREV = next++; AddPermanent(Format::RGBA16_SFLOAT); }
    if (hasDiff) { P_DIFF_ILLUM_PREV = next++; AddPermanent(Format::RGBA16_SFLOAT); }
    if (hasSpec) { P_SPEC_ILLUM_RESPONSIVE_PREV = next++; AddPermanent(Format::RGBA16_SFLOAT); }
    if (hasDiff) { P_DIFF_ILLUM_RESPONSIVE_PREV = next++; AddPermanent(Format::RGBA16_SFLOAT); }
    if (hasSpec)
    {
        P_REFLECTION_HIT_T_CURR = next++; P_REFLECTION_HIT_T_PREV = next++;
        AddPermanent(Format::R16_SFLOAT); AddPermanent(Format::R16_SFLOAT);
    }
    const uint16_t P_HISTORY_LENGTH_PREV = next++, P_NORMAL_ROUGHNESS_PREV = next++, P_MATERIAL_ID_PREV = next++, P_VIEWZ_PREV = next++;
    AddPermanent(Format::R8_UNORM);
    AddPermanent(Format::RGBA8_UNORM);
    AddPermanent(Format::R8_UNORM);
    AddPermanent(Format::R32_SFLOAT);

    next = kTransientBase;
    uint16_t T_SPEC_ILLUM_PING = 0, T_SPEC_ILLUM_PONG = 0, T_DIFF_ILLUM_PING = 0, T_DIFF_ILLUM_PONG = 0, T_SPEC_REPROJECTION_CONFIDENCE = 0;
    if (hasSpec) { T_SPEC_ILLUM_PING = next++; T_SPEC_ILLUM_PONG = next++; AddTransient(Format::RGBA16_SFLOAT); AddTransient(Format::RGBA16_SFLOAT); }
    if (hasDiff) { T_DIFF_ILLUM_PING = next++; T_DIFF_ILLUM_PONG = next++; AddTransient(Format::RGBA16_SFLOAT); AddTransient(Format::RGBA16_SFLOAT); }
    if (hasSpec) { T_SPEC_REPROJECTION_CONFIDENCE = next++; AddTransient(Format::R8_UNORM); }
    const uint16_t T_TILES = next++, T_HISTORY_LENGTH = next++;
    AddTransient(Format::R8_UNORM, 16);
    AddTransient(Format::R8_UNORM);

    const uint16_t IN_SPEC = R(ResourceType::IN_SPEC_RADIANCE_HITDIST), IN_DIFF = R(ResourceType::IN_DIFF_RADIANCE_HITDIST);
    const uint16_t OUT_SPEC = R(ResourceType::OUT_SPEC_RADIANCE_HITDIST), OUT_DIFF = R(ResourceType::OUT_DIFF_RADIANCE_HITDIST);
    const uint16_t NR = R(ResourceType::IN_NORMAL_ROUGHNESS), VZ = R(ResourceType::IN_VIEWZ);
    // bindings of a signal that the denoiser does not have are simply not pushed
    auto InS = [&](uint16_t r, uint16_t swapWith = kNoSwap) { if (hasSpec) In(r, swapWith); };
    auto InD = [&](uint16_t r) { if (hasDiff) In(r); };
    auto OutS = [&](uint16_t r, uint16_t swapWith = kNoSwap) { if (hasSpec) Out(r, swapWith); };
    auto OutD = [&](uint16_t r) { if (hasDiff) Out(r); };

    BeginPass(dn, "Classify tiles");
    In(VZ);
    Out(T_TILES);
    Emit({Family::RELAX, Pass::ClassifyTiles}, 16, 16, cb); // shared by the three RELAX denoisers

    for (int i = 0; i < 2; i++)
    {
        BeginPass(dn, "Hit distance reconstruction");
        In(T_TILES); InS(IN_SPEC); InD(IN_DIFF); In(NR); In(VZ);
        OutS(T_SPEC_ILLUM_PING); OutD(T_DIFF_ILLUM_PING);
        Emit({Family::RELAX, i ? Pass::HitDistReconstruction_5x5 : Pass::HitDistReconstruction, signals}, 8, 8, cb);
    }

    for (int i = 0; i < 2; i++)
    {
        BeginPass(dn, "Pre-pass");
        In(T_TILES); InS(i ? T_SPEC_ILLUM_PING : IN_SPEC); InD(i ? T_DIFF_ILLUM_PING : IN_DIFF); In(NR); In(VZ);
        OutS(OUT_SPEC); OutD(OUT_DIFF);
        Emit({Family::RELAX, Pass::PrePass, signals}, 16, 16, cb);
    }

    for (int i = 0; i < 4; i++)
    {
        const bool hasMix = (i >> 1) & 1, hasConfidence = i & 1;
        BeginPass(dn, "Temporal accumulation");
        In(T_TILES); InS(OUT_SPEC); InD(OUT_DIFF); In(R(ResourceType::IN_MV)); In(NR); In(VZ);
        InS(P_SPEC_ILLUM_RESPONSIVE_PREV); InD(P_DIFF_ILLUM_RESPONSIVE_PREV); InS(P_SPEC_ILLUM_PREV); InD(P_DIFF_ILLUM_PREV);
        In(P_NORMAL_ROUGHNESS_PREV); In(P_VIEWZ_PREV); InS(P_REFLECTION_HIT_T_PREV, P_REFLECTION_HIT_T_CURR);
        In(P_HISTORY_LENGTH_PREV); In(P_MATERIAL_ID_PREV);
        InS(hasConfidence ? R(ResourceType::IN_SPEC_CONFIDENCE) : kDummy);
        InD(hasConfidence ? R(ResourceType::IN_DIFF_CONFIDENCE) : kDummy);
        In(hasMix ? R(ResourceType::IN_DISOCCLUSION_THRESHOLD_MIX) : kDummy);
        OutS(T_SPEC_ILLUM_PING); OutD(T_DIFF_ILLUM_PING); OutS(T_SPEC_ILLUM_PONG); OutD(T_DIFF_ILLUM_PONG);
        OutS(P_REFLECTION_HIT_T_CURR, P_REFLECTION_HIT_T_PREV); Out(T_HISTORY_LENGTH); OutS(T_SPEC_REPROJECTION_CONFIDENCE);
        Emit({Family::RELAX, Pass::TemporalAccumulation, signals}, 8, 16, cb);
    }

    BeginPass(dn, "History fix");
    In(T_TILES); InS(T_SPEC_ILLUM_PING); InD(T_DIFF_ILLUM_PING); In(T_HISTORY_LENGTH); In(NR); In(VZ);
    OutS(T_SPEC_ILLUM_PONG); OutD(T_DIFF_ILLUM_PONG);
    Emit({Family::RELAX, Pass::HistoryFix, signals}, 8, 8, cb);

    BeginPass(dn, "History clamping");
    In(T_TILES); In(VZ); InS(OUT_SPEC); InD(OUT_DIFF); InS(T_SPEC_ILLUM_PING); InD(T_DIFF_ILLUM_PING); InS(T_SPEC_ILLUM_PONG); InD(T_DIFF_ILLUM_PONG); In(T_HISTORY_LENGTH);
    OutS(P_SPEC_ILLUM_PREV); OutD(P_DIFF_ILLUM_PREV); OutS(P_SPEC_ILLUM_RESPONSIVE_PREV); OutD(P_DIFF_ILLUM_RESPONSIVE_PREV); Out(P_HISTORY_LENGTH_PREV);
    Emit({Family::RELAX, Pass::HistoryClamping, signals}, 8, 8, cb);

    BeginPass(dn, "Copy");
    InS(P_SPEC_ILLUM_PREV); InD(P_DIFF_ILLUM_PREV);
    OutS(OUT_SPEC); OutD(OUT_DIFF);
    Emit({Family::RELAX, Pass::Copy, signals}, 8, 8, cb);

    BeginPass(dn, "Anti-firefly");
    In(T_TILES); InS(OUT_SPEC); InD(OUT_DIFF); In(NR); In(VZ);
    OutS(P_SPEC_ILLUM_PREV); OutD(P_DIFF_ILLUM_PREV);
    Emit({Family::RELAX, Pass::AntiFirefly, signals}, 8, 8, cb);

    for (int i = 0; i < 2; i++)
    {
        const bool hasConfidence = i & 1;
        for (uint32_t j = 0; j < kAtrousBindingVariants; j++)
        {
            const bool isSmem = j == 0, isEven = (j % 2) == 0, isLast = j > 2;
            BeginPass(dn, isSmem ? "A-trous (SMEM)" : "A-trous");
            In(T_TILES);
            if (isSmem) { InS(P_SPEC_ILLUM_PREV); InD(P_DIFF_ILLUM_PREV); }
            else { InS(isEven ? T_SPEC_ILLUM_PONG : T_SPEC_ILLUM_PING); InD(isEven ? T_DIFF_ILLUM_PONG : T_DIFF_ILLUM_PING); }
            In(T_HISTORY_LENGTH); InS(T_SPEC_REPROJECTION_CONFIDENCE); In(NR); In(VZ);
            InS(hasConfidence ? R(ResourceType::IN_SPEC_CONFIDENCE) : kDummy);
            InD(hasConfidence ? R(ResourceType::IN_DIFF_CONFIDENCE) : kDummy);
            if (isLast) { OutS(OUT_SPEC); OutD(OUT_DIFF); }
            else { OutS(isEven ? T_SPEC_ILLUM_PING : T_SPEC_ILLUM_PONG); OutD(isEven ? T_DIFF_ILLUM_PING : T_DIFF_ILLUM_PONG); }
            if (isSmem) { Out(P_NORMAL_ROUGHNESS_PREV); Out(P_MATERIAL_ID_PREV); Out(P_VIEWZ_PREV); }
            const uint16_t repeats = isLast ? 1 : (kMaxAtrousPasses - 2 + 1) / 2;
            if (isSmem) Emit({Family::RELAX, Pass::AtrousSmem, signals}, 8, 8, cbAtrous);
            else Emit({Family::RELAX, Pass::Atrous, signals}, 16, 16, cbAtrous, 1, repeats);
        }
    }

    BeginPass(dn, "Split screen");
    In(VZ); InD(IN_DIFF); InS(IN_SPEC);
    OutD(OUT_DIFF); OutS(OUT_SPEC);
    Emit({Family::RELAX, Pass::SplitScreen, signals}, 8, 16, cb);

    BeginPass(dn, "Validation");
    In(NR); In(VZ); In(R(ResourceType::IN_MV)); In(T_HISTORY_LENGTH);
    Out(R(ResourceType::OUT_VALIDATION));
    Emit({Family::RELAX, Pass::Validation}, 8, 16, cb, kIgnoreRect);
}

void Scheduler::UpdateRelax(const DenoiserSlot& slot)
{
    const RelaxSettings& s = slot.settings.relax;
    const bool reconstruct = s.hitDistanceReconstructionMode != HitDistanceReconstructionMode::OFF && s.checkerboardMode == CheckerboardMode::OFF;
    const uint32_t iterations = std::min(std::max(s.atrousIterationNum, 2u), kMaxAtrousPasses);
    auto push = [&](uint32_t pass) { FillRelaxConstants(s, Push(slot, pass)); };

    if (common_.splitScreen >= 1.0f)
    {
        push(RX_SPLIT_SCREEN);
        return;
    }
    push(RX_CLASSIFY_TILES);
    if (reconstruct) push(RX_HITDIST_RECONSTRUCTION + (s.hitDistanceReconstructionMode == HitDistanceReconstructionMode::AREA_5X5 ? 1 : 0));
    push(RX_PREPASS + (reconstruct ? 1 : 0));
    push(RX_TEMPORAL_ACCUMULATION + (common_.isDisocclusionThresholdMixAvailable ? 2 : 0) + (common_.isHistoryConfidenceAvailable ? 1 : 0));
    push(RX_HISTORY_FIX);
    push(RX_HISTORY_CLAMPING);
    if (s.enableAntiFirefly)
    {
        push(RX_COPY);
        push(RX_ANTI_FIREFLY);
    }
    for (uint32_t i = 0; i < iterations; i++)
    {
        // binding variants: 0 = SMEM first pass, 1/2 = odd/even ping-pong, +2 = last pass writes the outputs
        uint32_t pass = RX_ATROUS + (common_.isHistoryConfidenceAvailable ? kAtrousBindingVariants : 0);
        if (i != 0) pass += 2 - (i & 1);
        if (i == iterations - 1) pass += 2;
        RelaxConstants* c = (RelaxConstants*)Push(slot, pass);
        FillRelaxConstants(s, c);
        if (c)
        {
            c->gStepSize = 1u << i;
            c->gIsLastPass = i == iterations - 1 ? 1 : 0;
        }
    }
    if (common_.splitScreen > 0.0f) push(RX_SPLIT_SCREEN);
    if (common_.enableValidation) push(RX_VALIDATION);
}

void Scheduler::FillRelaxConstants(const RelaxSettings& s, void* data)
{
    if (!data) return;
    // only the shared 704 bytes are written here; the block handed out by Push() is already zeroed
    RelaxConstants& c = *(RelaxConstants*)data;
    const CommonSettings& cs = common_;
    const float rectW = cs.rectSize[0], rectH = cs.rectSize[1];
    const float resW = cs.resourceSize[0], resH = cs.resourceSize[1];

    auto set4 = [](float* d, float x, float y, float z, float w) { d[0] = x; d[1] = y; d[2] = z; d[3] = w; };
    auto set2 = [](float* d, float x, float y) { d[0] = x; d[1] = y; };
    auto saturate = [](float x) { return std::min(std::max(x, 0.0f), 1.0f); };

    // world-space frustum axes: pixel ray = forward + right * (u*2-1) + up * (1-v*2)  (Relax.cpp:53-78)
    auto frustumAxes = [&](const Mat4& v2c, const Mat4& w2v, const Mat4& v2w, const float fr[4], float* right, float* up, float* fwd)
    {
        const float tanHalfFov = 1.0f / v2c.at(0, 0);
        const float aspect = v2c.at(0, 0) / v2c.at(1, 1);
        set4(right, w2v.at(0, 0) * tanHalfFov, w2v.at(0, 1) * tanHalfFov, w2v.at(0, 2) * tanHalfFov, 0.0f);
        set4(up, w2v.at(1, 0) * tanHalfFov * aspect, w2v.at(1, 1) * tanHalfFov * aspect, w2v.at(1, 2) * tanHalfFov * aspect, 0.0f);
        Vec4 f = v2w.mul({0.5f * fr[2] + fr[0], 0.5f * fr[3] + fr[1], 1.0f, 0.0f});
        set4(fwd, f.x, f.y, f.z, 0.0f);
    };

    memcpy(c.gWorldToClip, worldToClip.m, 64);
    memcpy(c.gWorldToClipPrev, worldToClipPrev.m, 64);
    memcpy(c.gWorldToViewPrev, worldToViewPrev.m, 64);
    memcpy(c.gWorldPrevToWorld, worldPrevToWorld.m, 64);
    set4(c.gRotatorPre, rotatorPre.x, rotatorPre.y, rotatorPre.z, rotatorPre.w);
    frustumAxes(viewToClip, worldToView, viewToWorld, frustum, c.gFrustumRight, c.gFrustumUp, c.gFrustumForward);
    frustumAxes(viewToClipPrev, worldToViewPrev, viewToWorldPrev, frustumPrev, c.gPrevFrustumRight, c.gPrevFrustumUp, c.gPrevFrustumForward);
    set4(c.gCameraDelta, cameraDelta.x, cameraDelta.y, cameraDelta.z, 0.0f);
    set4(c.gMvScale, cs.motionVectorScale[0], cs.motionVectorScale[1], cs.motionVectorScale[2], cs.isMotionVectorInWorldSpace ? 1.0f : 0.0f);
    set2(c.gJitter, cs.cameraJitter[0], cs.cameraJitter[1]);
    set2(c.gResolutionScale, rectW / resW, rectH / resH);
    set2(c.gRectOffset, float(cs.rectOrigin[0]) / resW, float(cs.rectOrigin[1]) / resH);
    set2(c.gResourceSizeInv, 1.0f / resW, 1.0f / resH);
    set2(c.gResourceSize, resW, resH);
    set2(c.gRectSizeInv, 1.0f / rectW, 1.0f / rectH);
    set2(c.gRectSizePrev, cs.rectSizePrev[0], cs.rectSizePrev[1]);
    set2(c.gResourceSizeInvPrev, 1.0f / float(cs.resourceSizePrev[0]), 1.0f / float(cs.resourceSizePrev[1]));
    c.gPrintfAt[0] = cs.printfAt[0]; c.gPrintfAt[1] = cs.printfAt[1];
    c.gRectOrigin[0] = cs.rectOrigin[0]; c.gRectOrigin[1] = cs.rectOrigin[1];
    c.gRectSize[0] = cs.rectSize[0]; c.gRectSize[1] = cs.rectSize[1];

    const bool reset = cs.accumulationMode != AccumulationMode::CONTINUE;
    const float bonus = (1.0f + jitterDelta) / rectH;
    c.gSpecMaxAccumulatedFrameNum = reset ? 0.0f : (float)std::min(s.specularMaxAccumulatedFrameNum, RELAX_MAX_HISTORY_FRAME_NUM);
    c.gSpecMaxFastAccumulatedFrameNum = reset ? 0.0f : (float)std::min(s.specularMaxFastAccumulatedFrameNum, RELAX_MAX_HISTORY_FRAME_NUM);
    c.gDiffMaxAccumulatedFrameNum = reset ? 0.0f : (float)std::min(s.diffuseMaxAccumulatedFrameNum, RELAX_MAX_HISTORY_FRAME_NUM);
    c.gDiffMaxFastAccumulatedFrameNum = reset ? 0.0f : (float)std::min(s.diffuseMaxFastAccumulatedFrameNum, RELAX_MAX_HISTORY_FRAME_NUM);
    c.gDisocclusionThreshold = cs.disocclusionThreshold + bonus;
    c.gDisocclusionThresholdAlternate = cs.disocclusionThresholdAlternate + bonus;
    c.gCameraAttachedReflectionMaterialID = cs.cameraAttachedReflectionMaterialID;
    c.gStrandMaterialID = cs.strandMaterialID;
    c.gStrandThickness = cs.strandThickness;
    c.gRoughnessFraction = s.roughnessFraction;
    c.gSpecVarianceBoost = s.specularVarianceBoost;
    c.gSplitScreen = cs.splitScreen;
    c.gDiffBlurRadius = s.diffusePrepassBlurRadius;
    c.gSpecBlurRadius = s.specularPrepassBlurRadius;
    c.gDepthThreshold = s.depthThreshold;
    c.gLobeAngleFraction = s.lobeAngleFraction;
    c.gSpecLobeAngleSlack = Radians(s.specularLobeAngleSlack);
    c.gHistoryFixEdgeStoppingNormalPower = s.historyFixEdgeStoppingNormalPower;
    c.gRoughnessEdgeStoppingRelaxation = s.roughnessEdgeStoppingRelaxation;
    c.gNormalEdgeStoppingRelaxation = s.normalEdgeStoppingRelaxation;
    c.gColorBoxSigmaScale = s.historyClampingColorBoxSigmaScale;
    c.gHistoryAccelerationAmount = s.antilagSettings.accelerationAmount;
    c.gHistoryResetTemporalSigmaScale = s.antilagSettings.temporalSigmaScale;
    c.gHistoryResetSpatialSigmaScale = s.antilagSettings.spatialSigmaScale;
    c.gHistoryResetAmount = s.antilagSettings.resetAmount;
    c.gDenoisingRange = cs.denoisingRange;
    c.gSpecPhiLuminance = s.specularPhiLuminance;
    c.gDiffPhiLuminance = s.diffusePhiLuminance;
    c.gDiffMaxLuminanceRelativeDifference = -std::log(saturate(s.diffuseMinLuminanceWeight));
    c.gSpecMaxLuminanceRelativeDifference = -std::log(saturate(s.specularMinLuminanceWeight));
    c.gLuminanceEdgeStoppingRelaxation = s.roughnessEdgeStoppingRelaxation; // sic: the reference reads the roughness setting here (Relax.cpp:156)
    c.gConfidenceDrivenRelaxationMultiplier = s.confidenceDrivenRelaxationMultiplier;
    c.gConfidenceDrivenLuminanceEdgeStoppingRelaxation = s.confidenceDrivenLuminanceEdgeStoppingRelaxation;
    c.gConfidenceDrivenNormalEdgeStoppingRelaxation = s.confidenceDrivenNormalEdgeStoppingRelaxation;
    c.gDebug = cs.debug;
    c.gOrthoMode = orthoMode;
    c.gUnproject = 1.0f / (0.5f * rectH * projectY);
    c.gFramerateScale = std::min(std::max(16.66f / timeDelta, 0.25f), 4.0f);
    c.gCheckerboardResolveAccumSpeed = checkerboardResolveAccumSpeed;
    c.gJitterDelta = jitterDelta;
    c.gHistoryFixFrameNum = s.historyFixFrameNum + 1.0f;
    c.gHistoryFixBasePixelStride = (float)s.historyFixBasePixelStride;
    c.gHistoryThreshold = (float)s.spatialVarianceEstimationHistoryThreshold;
    c.gViewZScale = cs.viewZScale;
    c.gMinHitDistanceWeight = s.minHitDistanceWeight * 2.0f;
    c.gDiffMinMaterial = s.minMaterialForDiffuse;
    c.gSpecMinMaterial = s.minMaterialForSpecular;
    c.gRoughnessEdgeStoppingEnabled = s.enableRoughnessEdgeStopping ? 1 : 0;
    c.gFrameIndex = cs.frameIndex;
    c.gDiffCheckerboard = s.checkerboardMode == CheckerboardMode::BLACK ? 0 : (s.checkerboardMode == CheckerboardMode::WHITE ? 1 : 2);
    c.gSpecCheckerboard = s.checkerboardMode == CheckerboardMode::BLACK ? 1 : (s.checkerboardMode == CheckerboardMode::WHITE ? 0 : 2);
    c.gHasHistoryConfidence = cs.isHistoryConfidenceAvailable ? 1 : 0;
    c.gHasDisocclusionThresholdMix = cs.isDisocclusionThresholdMixAvailable ? 1 : 0;
    c.gResetHistory = reset ? 1 : 0;
}
} // namespace nrdb200
