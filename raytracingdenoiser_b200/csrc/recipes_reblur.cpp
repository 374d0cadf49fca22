// REBLUR pass graphs and per-frame schedule.
// Restates (with one generic builder instead of three copies) the reference's
//   Source/Denoisers/Reblur_Diffuse.hpp, Reblur_Specular.hpp, Reblur_DiffuseSpecular.hpp   (pools, bindings, pass order)
//   Source/Reblur.cpp:104-210 (Update_Reblur: permutation choice), :297-406 (AddSharedConstants_Reblur)
// Binding order inside a pass is the order of the reference's *.resources.hlsli: all inputs, then all outputs.
#include "scheduler.h"

#include <algorithm>

using namespace nrd;

namespace nrdb200
{
namespace
{
constexpr uint16_t R(ResourceType t) { return (uint16_t)t; }
constexpr uint16_t kDummy = R(ResourceType::IN_VIEWZ); // absent optional inputs are bound to IN_VIEWZ (Reblur.cpp:67)

// local pass-table layout; every pass has a "performance mode" twin right after it (Reblur.cpp:106-118)
enum ReblurPass : uint32_t
{
    RB_CLASSIFY_TILES = 0,
    RB_HITDIST_RECONSTRUCTION = RB_CLASSIFY_TILES + 1,        // 4 permutations x 2
    RB_PREPASS = RB_HITDIST_RECONSTRUCTION + 4 * 2,           // 2 x 2
    RB_TEMPORAL_ACCUMULATION = RB_PREPASS + 2 * 2,            // 8 x 2
    RB_HISTORY_FIX = RB_TEMPORAL_ACCUMULATION + 8 * 2,        // 1 x 2
    RB_BLUR = RB_HISTORY_FIX + 2,                             // 1 x 2
    RB_POST_BLUR = RB_BLUR + 2,                               // 2 x 2
    RB_TEMPORAL_STABILIZATION = RB_POST_BLUR + 2 * 2,         // 2 x 2
    RB_SPLIT_SCREEN = RB_TEMPORAL_STABILIZATION + 2 * 2,
    RB_VALIDATION = RB_SPLIT_SCREEN + 1,
};

} // namespace

void Scheduler::AddReblur(DenoiserSlot& slot, bool hasDiff, bool hasSpec)
{
    new (&slot.settings.reblur) ReblurSettings();
    slot.settingsSize = sizeof(ReblurSettings);

    const uint8_t signals = (hasDiff ? SIGNAL_DIFFUSE : 0) | (hasSpec ? SIGNAL_SPECULAR : 0);
    const char* denoiserName = hasDiff && hasSpec ? "REBLUR_DiffuseSpecular" : (hasSpec ? "REBLUR_Specular" : "REBLUR_Diffuse");
    const uint32_t cb = sizeof(ReblurConstants);
    // a pass and its performance-mode twin
    auto EmitPair = [&](Pass pass) {
        Emit({Family::REBLUR, pass, signals}, 8, 16, cb);
        Emit({Family::REBLUR, pass, signals, true}, 8, 16, cb);
    };

    // ---- permanent pool (Reblur_DiffuseSpecular.hpp:22-51, Reblur_Diffuse.hpp:20-37, Reblur_Specular.hpp:20-45)
    uint16_t next = kPermanentBase;
    const uint16_t P_PREV_VIEWZ = next++;
    const uint16_t P_PREV_NORMAL_ROUGHNESS = next++;
    const uint16_t P_PREV_INTERNAL_DATA = next++;
    AddPermanent(Format::R32_SFLOAT);
    AddPermanent(Format::R10_G10_B10_A2_UNORM);
    AddPermanent(Format::R16_UINT);
    uint16_t P_DIFF_HISTORY = 0, P_DIFF_FAST = 0, P_DIFF_STAB_PING = 0, P_DIFF_STAB_PONG = 0;
    uint16_t P_SPEC_HISTORY = 0, P_SPEC_FAST = 0, P_SPEC_STAB_PING = 0, P_SPEC_STAB_PONG = 0, P_HITDIST_PING = 0, P_HITDIST_PONG = 0;
    if (hasDiff)
    {
        P_DIFF_HISTORY = next++; P_DIFF_FAST = next++; P_DIFF_STAB_PING = next++; P_DIFF_STAB_PONG = next++;
        AddPermanent(Format::RGBA16_SFLOAT); AddPermanent(Format::R16_SFLOAT); AddPermanent(Format::R16_SFLOAT); AddPermanent(Format::R16_SFLOAT);
    }
    if (hasSpec)
    {
        P_SPEC_HISTORY = next++; P_SPEC_FAST = next++; P_SPEC_STAB_PING = next++; P_SPEC_STAB_PONG = next++;
        AddPermanent(Format::RGBA16_SFLOAT); AddPermanent(Format::R16_SFLOAT); AddPermanent(Format::R16_SFLOAT); AddPermanent(Format::R16_SFLOAT);
        P_HITDIST_PING = next++; P_HITDIST_PONG = next++;
        AddPermanent(Format::R16_SFLOAT); AddPermanent(Format::R16_SFLOAT);
    }

    // ---- transient pool (Reblur_DiffuseSpecular.hpp:53-72, Reblur_Diffuse.hpp:39-52, Reblur_Specular.hpp:47-60)
    next = kTransientBase;
    const uint16_t T_DATA1 = next++;
    const uint16_t T_DATA2 = next++;
    AddTransient(hasDiff && hasSpec ? Format::RG8_UNORM : Format::R8_UNORM);
    AddTransient(hasSpec ? Format::R32_UINT : Format::R8_UINT);
    uint16_t T_HITDIST = 0, T_DIFF_TMP2 = 0, T_DIFF_FAST = 0, T_SPEC_TMP2 = 0, T_SPEC_FAST = 0;
    if (hasSpec) { T_HITDIST = next++; AddTransient(Format::R16_SFLOAT); }
    if (hasDiff) { T_DIFF_TMP2 = next++; T_DIFF_FAST = next++; AddTransient(Format::RGBA16_SFLOAT); AddTransient(Format::R16_SFLOAT); }
    if (hasSpec) { T_SPEC_TMP2 = next++; T_SPEC_FAST = next++; AddTransient(Format::RGBA16_SFLOAT); AddTransient(Format::R16_SFLOAT); }
    const uint16_t T_TILES = next++;
    AddTransient(Format::R8_UNORM, 16);

    // the application's outputs double as scratch (Reblur_DiffuseSpecular.hpp:14-17)
    const uint16_t DIFF_TEMP1 = R(ResourceType::OUT_DIFF_RADIANCE_HITDIST), DIFF_TEMP2 = T_DIFF_TMP2;
    const uint16_t SPEC_TEMP1 = R(ResourceType::OUT_SPEC_RADIANCE_HITDIST), SPEC_TEMP2 = T_SPEC_TMP2;
    const uint16_t IN_DIFF = R(ResourceType::IN_DIFF_RADIANCE_HITDIST), IN_SPEC = R(ResourceType::IN_SPEC_RADIANCE_HITDIST);

    BeginPass(denoiserName, "Classify tiles");
    In(R(ResourceType::IN_VIEWZ));
    Out(T_TILES);
    Emit({Family::REBLUR, Pass::ClassifyTiles}, 16, 16, cb); // shared by the three REBLUR denoisers

    for (int i = 0; i < 4; i++)
    {
        const bool is5x5 = (i >> 1) & 1, prepassEnabled = i & 1;
        BeginPass(denoiserName, "Hit distance reconstruction");
        In(T_TILES); In(R(ResourceType::IN_NORMAL_ROUGHNESS)); In(R(ResourceType::IN_VIEWZ));
        if (hasDiff) In(IN_DIFF);
        if (hasSpec) In(IN_SPEC);
        if (hasDiff) Out(prepassEnabled ? DIFF_TEMP2 : DIFF_TEMP1);
        if (hasSpec) Out(prepassEnabled ? SPEC_TEMP2 : SPEC_TEMP1);
        EmitPair(is5x5 ? Pass::HitDistReconstruction_5x5 : Pass::HitDistReconstruction);
    }

    for (int i = 0; i < 2; i++)
    {
        const bool afterReconstruction = i & 1;
        BeginPass(denoiserName, "Pre-pass");
        In(T_TILES); In(R(ResourceType::IN_NORMAL_ROUGHNESS)); In(R(ResourceType::IN_VIEWZ));
        if (hasDiff) In(afterReconstruction ? DIFF_TEMP2 : IN_DIFF);
        if (hasSpec) In(afterReconstruction ? SPEC_TEMP2 : IN_SPEC);
        if (hasDiff) Out(DIFF_TEMP1);
        if (hasSpec) { Out(SPEC_TEMP1); Out(T_HITDIST); }
        EmitPair(Pass::PrePass);
    }

    for (int i = 0; i < 8; i++)
    {
        const bool hasMix = (i >> 2) & 1, hasConfidence = (i >> 1) & 1, afterPrepass = i & 1;
        BeginPass(denoiserName, "Temporal accumulation");
        In(T_TILES); In(R(ResourceType::IN_NORMAL_ROUGHNESS)); In(R(ResourceType::IN_VIEWZ)); In(R(ResourceType::IN_MV));
        In(P_PREV_VIEWZ); In(P_PREV_NORMAL_ROUGHNESS); In(P_PREV_INTERNAL_DATA);
        In(hasMix ? R(ResourceType::IN_DISOCCLUSION_THRESHOLD_MIX) : kDummy);
        if (hasDiff) In(hasConfidence ? R(ResourceType::IN_DIFF_CONFIDENCE) : kDummy);
        if (hasSpec) In(hasConfidence ? R(ResourceType::IN_SPEC_CONFIDENCE) : kDummy);
        if (hasDiff) In(afterPrepass ? DIFF_TEMP1 : IN_DIFF);
        if (hasSpec) In(afterPrepass ? SPEC_TEMP1 : IN_SPEC);
        if (hasDiff && hasSpec) { In(P_DIFF_HISTORY); In(P_SPEC_HISTORY); In(P_DIFF_FAST); In(P_SPEC_FAST); }
        else if (hasDiff) { In(P_DIFF_HISTORY); In(P_DIFF_FAST); }
        else { In(P_SPEC_HISTORY); In(P_SPEC_FAST); }
        if (hasSpec) { In(P_HITDIST_PING, P_HITDIST_PONG); In(T_HITDIST); }
        if (hasDiff) Out(DIFF_TEMP2);
        if (hasSpec) Out(SPEC_TEMP2);
        if (hasDiff) Out(T_DIFF_FAST);
        if (hasSpec) { Out(T_SPEC_FAST); Out(P_HITDIST_PONG, P_HITDIST_PING); }
        Out(T_DATA1); Out(T_DATA2);
        EmitPair(Pass::TemporalAccumulation);
    }

    BeginPass(denoiserName, "History fix");
    In(T_TILES); In(R(ResourceType::IN_NORMAL_ROUGHNESS)); In(T_DATA1); In(R(ResourceType::IN_VIEWZ));
    if (hasDiff) In(DIFF_TEMP2);
    if (hasSpec) In(SPEC_TEMP2);
    if (hasDiff) In(T_DIFF_FAST);
    if (hasSpec) In(T_SPEC_FAST);
    if (hasDiff) Out(DIFF_TEMP1);
    if (hasSpec) Out(SPEC_TEMP1);
    if (hasDiff) Out(P_DIFF_FAST);
    if (hasSpec) Out(P_SPEC_FAST);
    EmitPair(Pass::HistoryFix);

    BeginPass(denoiserName, "Blur");
    In(T_TILES); In(R(ResourceType::IN_NORMAL_ROUGHNESS)); In(T_DATA1);
    if (hasDiff) In(DIFF_TEMP1);
    if (hasSpec) In(SPEC_TEMP1);
    In(R(ResourceType::IN_VIEWZ));
    if (hasDiff) Out(DIFF_TEMP2);
    if (hasSpec) Out(SPEC_TEMP2);
    Out(P_PREV_VIEWZ);
    EmitPair(Pass::Blur);

    for (int i = 0; i < 2; i++)
    {
        const bool withStabilization = i & 1;
        BeginPass(denoiserName, "Post-blur");
        In(T_TILES); In(R(ResourceType::IN_NORMAL_ROUGHNESS)); In(T_DATA1);
        if (hasDiff) In(DIFF_TEMP2);
        if (hasSpec) In(SPEC_TEMP2);
        In(P_PREV_VIEWZ);
        Out(P_PREV_NORMAL_ROUGHNESS);
        if (hasDiff) Out(P_DIFF_HISTORY);
        if (hasSpec) Out(P_SPEC_HISTORY);
        if (!withStabilization)
        {
            Out(P_PREV_INTERNAL_DATA);
            if (hasDiff) Out(R(ResourceType::OUT_DIFF_RADIANCE_HITDIST));
            if (hasSpec) Out(R(ResourceType::OUT_SPEC_RADIANCE_HITDIST));
        }
        EmitPair(withStabilization ? Pass::PostBlur : Pass::PostBlur_NoTemporalStabilization);
    }

    for (int i = 0; i < 2; i++)
    {
        const bool hasBaseColor = i & 1;
        BeginPass(denoiserName, "Temporal stabilization");
        In(T_TILES); In(R(ResourceType::IN_NORMAL_ROUGHNESS));
        if (hasSpec) In(hasBaseColor ? R(ResourceType::IN_BASECOLOR_METALNESS) : kDummy);
        In(P_PREV_VIEWZ); In(T_DATA1); In(T_DATA2);
        if (hasDiff) In(P_DIFF_HISTORY);
        if (hasSpec) In(P_SPEC_HISTORY);
        if (hasDiff) In(P_DIFF_STAB_PING, P_DIFF_STAB_PONG);
        if (hasSpec) { In(P_SPEC_STAB_PING, P_SPEC_STAB_PONG); In(P_HITDIST_PONG, P_HITDIST_PING); }
        Out(R(ResourceType::IN_MV)); // bound as storage: the pass may patch motion vectors
        Out(P_PREV_INTERNAL_DATA);
        if (hasDiff) Out(R(ResourceType::OUT_DIFF_RADIANCE_HITDIST));
        if (hasSpec) Out(R(ResourceType::OUT_SPEC_RADIANCE_HITDIST));
        if (hasDiff) Out(P_DIFF_STAB_PONG, P_DIFF_STAB_PING);
        if (hasSpec) Out(P_SPEC_STAB_PONG, P_SPEC_STAB_PING);
        EmitPair(Pass::TemporalStabilization);
    }

    BeginPass(denoiserName, "Split screen");
    In(R(ResourceType::IN_VIEWZ));
    if (hasDiff) In(IN_DIFF);
    if (hasSpec) In(IN_SPEC);
    if (hasDiff) Out(R(ResourceType::OUT_DIFF_RADIANCE_HITDIST));
    if (hasSpec) Out(R(ResourceType::OUT_SPEC_RADIANCE_HITDIST));
    Emit({Family::REBLUR, Pass::SplitScreen, signals}, 8, 16, cb);

    BeginPass(denoiserName, "Validation");
    In(R(ResourceType::IN_NORMAL_ROUGHNESS)); In(R(ResourceType::IN_VIEWZ)); In(R(ResourceType::IN_MV)); In(T_DATA1); In(T_DATA2);
    // a one-signal denoiser binds its only signal in both slots (Denoisers/Reblur_Diffuse.hpp, Reblur_Specular.hpp: REBLUR_ADD_VALIDATION_DISPATCH)
    In(hasDiff ? IN_DIFF : IN_SPEC);
    In(hasSpec ? IN_SPEC : IN_DIFF);
    Out(R(ResourceType::OUT_VALIDATION));
    Emit({Family::REBLUR, Pass::Validation}, 8, 16, cb + 8, kIgnoreRect); // + gHasDiffuse, gHasSpecular (840 = sizeof of the reference struct)
}

void Scheduler::UpdateReblur(const DenoiserSlot& slot)
{
    const ReblurSettings& s = slot.settings.reblur;
    const bool hasDiff = slot.desc.denoiser != Denoiser::REBLUR_SPECULAR;
    const bool hasSpec = slot.desc.denoiser != Denoiser::REBLUR_DIFFUSE;
    const uint32_t perf = s.enablePerformanceMode ? 1 : 0;

    const bool reconstruct = s.hitDistanceReconstructionMode != HitDistanceReconstructionMode::OFF && s.checkerboardMode == CheckerboardMode::OFF;
    const bool skipStabilization = s.maxStabilizedFrameNum == 0;
    const bool skipPrePass = (s.diffusePrepassBlurRadius == 0.0f || !hasDiff) && (s.specularPrepassBlurRadius == 0.0f || !hasSpec) &&
                             s.checkerboardMode == CheckerboardMode::OFF;

    auto push = [&](uint32_t pass) { FillReblurConstants(s, Push(slot, pass)); };

    if (common_.splitScreen >= 1.0f)
    {
        push(RB_SPLIT_SCREEN);
        return;
    }

    push(RB_CLASSIFY_TILES);
    if (reconstruct)
        push(RB_HITDIST_RECONSTRUCTION + (s.hitDistanceReconstructionMode == HitDistanceReconstructionMode::AREA_5X5 ? 4 : 0) + (!skipPrePass ? 2 : 0) + perf);
    if (!skipPrePass)
        push(RB_PREPASS + (reconstruct ? 2 : 0) + perf);
    push(RB_TEMPORAL_ACCUMULATION + (common_.isDisocclusionThresholdMixAvailable ? 8 : 0) + (common_.isHistoryConfidenceAvailable ? 4 : 0) +
         ((!skipPrePass || reconstruct) ? 2 : 0) + perf);
    push(RB_HISTORY_FIX + perf);
    push(RB_BLUR + perf);
    push(RB_POST_BLUR + (skipStabilization ? 0 : 2) + perf);
    if (!skipStabilization)
        push(RB_TEMPORAL_STABILIZATION + (common_.isBaseColorMetalnessAvailable ? 2 : 0) + perf);
    if (common_.splitScreen > 0.0f)
        push(RB_SPLIT_SCREEN);
    if (common_.enableValidation)
    {
        uint8_t* c = (uint8_t*)Push(slot, RB_VALIDATION);
        FillReblurConstants(s, c);
        uint32_t extra[2] = {hasDiff ? 1u : 0u, hasSpec ? 1u : 0u};
        memcpy(c + sizeof(ReblurConstants), extra, sizeof(extra));
    }
}

void Scheduler::FillReblurConstants(const ReblurSettings& s, void* data)
{
    if (!data) return;
    ReblurConstants& c = *(ReblurConstants*)data;
    const CommonSettings& cs = common_;
    const float rectW = cs.rectSize[0], rectH = cs.rectSize[1], rectWprev = cs.rectSizePrev[0], rectHprev = cs.rectSizePrev[1];
    const float resW = cs.resourceSize[0], resH = cs.resourceSize[1], resWprev = cs.resourceSizePrev[0], resHprev = cs.resourceSizePrev[1];

    const bool isRectChanged = cs.rectSize[0] != cs.rectSizePrev[0] || cs.rectSize[1] != cs.rectSizePrev[1];
    const bool isHistoryReset = cs.accumulationMode != AccumulationMode::CONTINUE;
    const float unproject = 1.0f / (0.5f * rectH * projectY);
    const float worstResolutionScale = std::min(rectW / resW, rectH / resH);
    const float maxBlurRadius = s.maxBlurRadius * worstResolutionScale;
    const float disocclusionBonus = (1.0f + jitterDelta) / rectH;
    const float stabilizationStrength = s.maxStabilizedFrameNum / (1.0f + s.maxStabilizedFrameNum);
    const float hitDistStabilizationStrength = s.maxStabilizedFrameNumForHitDistance / (1.0f + s.maxStabilizedFrameNumForHitDistance);
    const uint32_t maxAccumulated = std::min(s.maxAccumulatedFrameNum, REBLUR_MAX_HISTORY_FRAME_NUM);

    uint32_t diffCheckerboard = 2, specCheckerboard = 2;
    if (s.checkerboardMode == CheckerboardMode::BLACK) { diffCheckerboard = 0; specCheckerboard = 1; }
    else if (s.checkerboardMode == CheckerboardMode::WHITE) { diffCheckerboard = 1; specCheckerboard = 0; }

    auto set4 = [](float* d, float x, float y, float z, float w) { d[0] = x; d[1] = y; d[2] = z; d[3] = w; };
    auto set2 = [](float* d, float x, float y) { d[0] = x; d[1] = y; };

    memcpy(c.gWorldToClip, worldToClip.m, 64);
    memcpy(c.gViewToClip, viewToClip.m, 64);
    memcpy(c.gViewToWorld, viewToWorld.m, 64);
    memcpy(c.gWorldToViewPrev, worldToViewPrev.m, 64);
    memcpy(c.gWorldToClipPrev, worldToClipPrev.m, 64);
    memcpy(c.gWorldPrevToWorld, worldPrevToWorld.m, 64);
    set4(c.gRotatorPre, rotatorPre.x, rotatorPre.y, rotatorPre.z, rotatorPre.w);
    set4(c.gRotator, rotator.x, rotator.y, rotator.z, rotator.w);
    set4(c.gRotatorPost, rotatorPost.x, rotatorPost.y, rotatorPost.z, rotatorPost.w);
    memcpy(c.gFrustum, frustum, 16);
    memcpy(c.gFrustumPrev, frustumPrev, 16);
    set4(c.gCameraDelta, cameraDelta.x, cameraDelta.y, cameraDelta.z, 0.0f);
    set4(c.gHitDistParams, s.hitDistanceParameters.A, s.hitDistanceParameters.B, s.hitDistanceParameters.C, s.hitDistanceParameters.D);
    set4(c.gViewVectorWorld, viewDirection.x, viewDirection.y, viewDirection.z, 0.0f);
    set4(c.gViewVectorWorldPrev, viewDirectionPrev.x, viewDirectionPrev.y, viewDirectionPrev.z, 0.0f);
    set4(c.gMvScale, cs.motionVectorScale[0], cs.motionVectorScale[1], cs.motionVectorScale[2], cs.isMotionVectorInWorldSpace ? 1.0f : 0.0f);
    set2(c.gAntilagParams, s.antilagSettings.luminanceSigmaScale, s.antilagSettings.luminanceSensitivity);
    set2(c.gResourceSize, resW, resH);
    set2(c.gResourceSizeInv, 1.0f / resW, 1.0f / resH);
    set2(c.gResourceSizeInvPrev, 1.0f / resWprev, 1.0f / resHprev);
    set2(c.gRectSize, rectW, rectH);
    set2(c.gRectSizeInv, 1.0f / rectW, 1.0f / rectH);
    set2(c.gRectSizePrev, rectWprev, rectHprev);
    set2(c.gResolutionScale, rectW / resW, rectH / resH);
    set2(c.gResolutionScalePrev, rectWprev / resWprev, rectHprev / resHprev);
    set2(c.gRectOffset, float(cs.rectOrigin[0]) / resW, float(cs.rectOrigin[1]) / resH);
    set2(c.gSpecProbabilityThresholdsForMvModification,
         cs.isBaseColorMetalnessAvailable ? s.specularProbabilityThresholdsForMvModification[0] : 2.0f,
         cs.isBaseColorMetalnessAvailable ? s.specularProbabilityThresholdsForMvModification[1] : 3.0f);
    set2(c.gJitter, cs.cameraJitter[0], cs.cameraJitter[1]);
    c.gPrintfAt[0] = cs.printfAt[0]; c.gPrintfAt[1] = cs.printfAt[1];
    c.gRectOrigin[0] = cs.rectOrigin[0]; c.gRectOrigin[1] = cs.rectOrigin[1];
    c.gRectSizeMinusOne[0] = cs.rectSize[0] - 1; c.gRectSizeMinusOne[1] = cs.rectSize[1] - 1;
    c.gDisocclusionThreshold = cs.disocclusionThreshold + disocclusionBonus;
    c.gDisocclusionThresholdAlternate = cs.disocclusionThresholdAlternate + disocclusionBonus;
    c.gCameraAttachedReflectionMaterialID = cs.cameraAttachedReflectionMaterialID;
    c.gStrandMaterialID = cs.strandMaterialID;
    c.gStrandThickness = cs.strandThickness;
    c.gStabilizationStrength = isHistoryReset ? 0.0f : stabilizationStrength;
    c.gHitDistStabilizationStrength = isHistoryReset ? 0.0f : hitDistStabilizationStrength;
    c.gDebug = cs.debug;
    c.gOrthoMode = orthoMode;
    c.gUnproject = unproject;
    c.gDenoisingRange = cs.denoisingRange;
    c.gPlaneDistSensitivity = s.planeDistanceSensitivity;
    c.gFramerateScale = frameRateScale;
    c.gMinBlurRadius = s.minBlurRadius;
    c.gMaxBlurRadius = std::max(maxBlurRadius, s.minBlurRadius);
    c.gDiffPrepassBlurRadius = s.diffusePrepassBlurRadius * worstResolutionScale;
    c.gSpecPrepassBlurRadius = s.specularPrepassBlurRadius * worstResolutionScale;
    c.gMaxAccumulatedFrameNum = isHistoryReset ? 0.0f : float(maxAccumulated);
    c.gMaxFastAccumulatedFrameNum = isHistoryReset ? 0.0f : float(s.maxFastAccumulatedFrameNum);
    c.gAntiFirefly = s.enableAntiFirefly ? 1.0f : 0.0f;
    c.gLobeAngleFraction = s.lobeAngleFraction * s.lobeAngleFraction; // squared on purpose (Reblur.cpp:384)
    c.gRoughnessFraction = s.roughnessFraction;
    c.gResponsiveAccumulationRoughnessThreshold = s.responsiveAccumulationRoughnessThreshold;
    c.gHistoryFixFrameNum = (float)s.historyFixFrameNum;
    c.gHistoryFixBasePixelStride = (float)s.historyFixBasePixelStride;
    c.gMinRectDimMulUnproject = std::min(rectW, rectH) * unproject;
    c.gUsePrepassNotOnlyForSpecularMotionEstimation = s.usePrepassOnlyForSpecularMotionEstimation ? 0.0f : 1.0f;
    c.gSplitScreen = cs.splitScreen;
    c.gSplitScreenPrev = splitScreenPrev;
    c.gCheckerboardResolveAccumSpeed = checkerboardResolveAccumSpeed;
    c.gViewZScale = cs.viewZScale;
    c.gFireflySuppressorMinRelativeScale = s.fireflySuppressorMinRelativeScale;
    c.gMinHitDistanceWeight = s.minHitDistanceWeight;
    c.gDiffMinMaterial = s.minMaterialForDiffuse;
    c.gSpecMinMaterial = s.minMaterialForSpecular;
    c.gHasHistoryConfidence = cs.isHistoryConfidenceAvailable ? 1 : 0;
    c.gHasDisocclusionThresholdMix = cs.isDisocclusionThresholdMixAvailable ? 1 : 0;
    c.gDiffCheckerboard = diffCheckerboard;
    c.gSpecCheckerboard = specCheckerboard;
    c.gFrameIndex = cs.frameIndex;
    c.gIsRectChanged = isRectChanged ? 1 : 0;
    c.gResetHistory = isHistoryReset ? 1 : 0;
}
} // namespace nrdb200
