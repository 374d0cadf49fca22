// SIGMA_SHADOW / SIGMA_SHADOW_TRANSLUCENCY pass graphs and per-frame schedule.
// Restates the reference's Source/Denoisers/Sigma_Shadow.hpp:11-170, Sigma_ShadowTranslucency.hpp:11-173 (pools, bindings) and
// Source/Sigma.cpp:25-90 (Update_SigmaShadow), :92-145 (AddSharedConstants_Sigma).
#include "scheduler.h"

#include <algorithm>
#include <cstring>

using namespace nrd;

namespace nrdb200
{
namespace
{
constexpr uint16_t R(ResourceType t) { return (uint16_t)t; }
enum SigmaPass : uint32_t { SG_CLASSIFY_TILES, SG_SMOOTH_TILES, SG_COPY, SG_BLUR, SG_POST_BLUR /* 2 */, SG_TEMPORAL_STABILIZATION = SG_POST_BLUR + 2, SG_SPLIT_SCREEN };
} // namespace

// translucent = SIGMA_SHADOW_TRANSLUCENCY: the shadow signal is a float4 (SIGMA_TYPE, SIGMA_Config.hlsli:38-43) in RGBA8 textures,
// IN_TRANSLUCENCY feeds ClassifyTiles / Blur / SplitScreen, and Blur runs at the rect size instead of USE_MAX_DIMS
void Scheduler::AddSigmaShadow(DenoiserSlot& slot, bool translucent)
{
    new (&slot.settings.sigma) SigmaSettings();
    slot.settingsSize = sizeof(SigmaSettings);
    const char* dn = translucent ? "SIGMA_ShadowTranslucency" : "SIGMA_Shadow";
    const Format shadowFormat = translucent ? Format::RGBA8_UNORM : Format::R8_UNORM;
    // "SIGMA_Shadow_<pass>.cs" / "SIGMA_ShadowTranslucency_<pass>.cs"; SmoothTiles and Copy are shared by both denoisers
    auto kind = [&](Pass pass) { return PassKind{Family::SIGMA, pass, SIGNAL_SHADOW, false, translucent}; };
    // the reference reports sizeof() of its C++ struct, which has no tail padding to a 16-byte register (516, not 528)
    const uint32_t cb = offsetof(SigmaConstants, gIsRectChanged) + sizeof(uint32_t);

    const uint16_t P_HISTORY_LENGTH = kPermanentBase;
    AddPermanent(Format::R32_UINT);

    const uint16_t T_DATA_1 = kTransientBase, T_DATA_2 = kTransientBase + 1, T_TEMP_1 = kTransientBase + 2, T_TEMP_2 = kTransientBase + 3,
                   T_HISTORY = kTransientBase + 4, T_HISTORY_LENGTH = kTransientBase + 5, T_TILES = kTransientBase + 6, T_SMOOTHED_TILES = kTransientBase + 7;
    AddTransient(Format::R16_SFLOAT);
    AddTransient(Format::R16_SFLOAT);
    AddTransient(shadowFormat);
    AddTransient(shadowFormat);
    AddTransient(shadowFormat);
    AddTransient(Format::R32_UINT);
    AddTransient(Format::RGBA8_UNORM, 16);
    AddTransient(Format::RG8_UNORM, 16);

    BeginPass(dn, "Classify tiles");
    In(R(ResourceType::IN_VIEWZ)); In(R(ResourceType::IN_PENUMBRA));
    if (translucent) In(R(ResourceType::IN_TRANSLUCENCY));
    Out(T_TILES);
    Emit(kind(Pass::ClassifyTiles), 16, 16, cb);

    BeginPass(dn, "Smooth tiles");
    In(T_TILES);
    Out(T_SMOOTHED_TILES);
    Emit({Family::SIGMA, Pass::SmoothTiles}, 16, 16, cb, 16);

    BeginPass(dn, "Copy");
    In(T_SMOOTHED_TILES); In(R(ResourceType::OUT_SHADOW_TRANSLUCENCY)); In(P_HISTORY_LENGTH);
    Out(T_HISTORY); Out(T_HISTORY_LENGTH);
    Emit({Family::SIGMA, Pass::Copy}, 8, 16, cb, kUseMaxDims);

    BeginPass(dn, "Blur");
    In(R(ResourceType::IN_VIEWZ)); In(R(ResourceType::IN_NORMAL_ROUGHNESS)); In(R(ResourceType::IN_PENUMBRA)); In(T_SMOOTHED_TILES);
    if (translucent) In(R(ResourceType::IN_TRANSLUCENCY));
    Out(T_DATA_1); Out(T_TEMP_1);
    Emit(kind(Pass::Blur), 8, 16, cb, translucent ? (uint16_t)1 : kUseMaxDims);

    for (int i = 0; i < 2; i++)
    {
        const bool stabilized = i & 1;
        BeginPass(dn, "Post-blur");
        In(R(ResourceType::IN_VIEWZ)); In(R(ResourceType::IN_NORMAL_ROUGHNESS)); In(T_DATA_1); In(T_SMOOTHED_TILES); In(T_TEMP_1);
        Out(T_DATA_2);
        Out(stabilized ? T_TEMP_2 : R(ResourceType::OUT_SHADOW_TRANSLUCENCY));
        Emit(kind(Pass::PostBlur), 8, 16, cb);
    }

    BeginPass(dn, "Temporal stabilization");
    In(R(ResourceType::IN_VIEWZ)); In(R(ResourceType::IN_MV)); In(T_DATA_2); In(T_TEMP_2); In(T_HISTORY); In(T_HISTORY_LENGTH); In(T_SMOOTHED_TILES);
    Out(R(ResourceType::OUT_SHADOW_TRANSLUCENCY)); Out(P_HISTORY_LENGTH);
    Emit(kind(Pass::TemporalStabilization), 8, 16, cb);

    BeginPass(dn, "Split screen");
    In(R(ResourceType::IN_VIEWZ)); In(R(ResourceType::IN_PENUMBRA));
    if (translucent) In(R(ResourceType::IN_TRANSLUCENCY));
    Out(R(ResourceType::OUT_SHADOW_TRANSLUCENCY));
    Emit(kind(Pass::SplitScreen), 8, 16, cb);
}

void Scheduler::UpdateSigma(const DenoiserSlot& slot)
{
    const SigmaSettings& s = slot.settings.sigma;
    auto push = [&](uint32_t pass) { FillSigmaConstants(s, Push(slot, pass)); };

    if (common_.splitScreen >= 1.0f)
    {
        push(SG_SPLIT_SCREEN);
        return;
    }
    push(SG_CLASSIFY_TILES);
    push(SG_SMOOTH_TILES);
    if (s.maxStabilizedFrameNum) push(SG_COPY);
    push(SG_BLUR);
    push(SG_POST_BLUR + (s.maxStabilizedFrameNum ? 1 : 0));
    if (s.maxStabilizedFrameNum) push(SG_TEMPORAL_STABILIZATION);
    if (common_.splitScreen > 0.0f) push(SG_SPLIT_SCREEN);
}

void Scheduler::FillSigmaConstants(const SigmaSettings& s, void* data)
{
    if (!data) return;
    SigmaConstants& c = *(SigmaConstants*)data;
    const CommonSettings& cs = common_;
    const float rectW = cs.rectSize[0], rectH = cs.rectSize[1];
    const float resW = cs.resourceSize[0], resH = cs.resourceSize[1];
    const float unproject = 1.0f / (0.5f * rectH * projectY);
    const uint32_t frameNum = std::min(s.maxStabilizedFrameNum, SIGMA_MAX_HISTORY_FRAME_NUM);
    const float stabilizationStrength = frameNum / (1.0f + frameNum);
    // light direction rotated into view space (direction, so no translation)
    const float* l = s.lightDirection;
    const float lv[3] = {worldToView.at(0, 0) * l[0] + worldToView.at(0, 1) * l[1] + worldToView.at(0, 2) * l[2],
                         worldToView.at(1, 0) * l[0] + worldToView.at(1, 1) * l[1] + worldToView.at(1, 2) * l[2],
                         worldToView.at(2, 0) * l[0] + worldToView.at(2, 1) * l[1] + worldToView.at(2, 2) * l[2]};

    auto set4 = [](float* d, float x, float y, float z, float w) { d[0] = x; d[1] = y; d[2] = z; d[3] = w; };
    auto set2 = [](float* d, float x, float y) { d[0] = x; d[1] = y; };

    memcpy(c.gWorldToView, worldToView.m, 64);
    memcpy(c.gViewToClip, viewToClip.m, 64);
    memcpy(c.gWorldToClipPrev, worldToClipPrev.m, 64);
    memcpy(c.gWorldToViewPrev, worldToViewPrev.m, 64);
    set4(c.gRotator, rotator.x, rotator.y, rotator.z, rotator.w);
    set4(c.gRotatorPost, rotatorPost.x, rotatorPost.y, rotatorPost.z, rotatorPost.w);
    set4(c.gViewVectorWorld, viewDirection.x, viewDirection.y, viewDirection.z, 0.0f);
    set4(c.gLightDirectionView, lv[0], lv[1], lv[2], 0.0f);
    memcpy(c.gFrustum, frustum, 16);
    memcpy(c.gFrustumPrev, frustumPrev, 16);
    set4(c.gCameraDelta, cameraDelta.x, cameraDelta.y, cameraDelta.z, 0.0f);
    set4(c.gMvScale, cs.motionVectorScale[0], cs.motionVectorScale[1], cs.motionVectorScale[2], cs.isMotionVectorInWorldSpace ? 1.0f : 0.0f);
    set2(c.gResourceSizeInv, 1.0f / resW, 1.0f / resH);
    set2(c.gResourceSizeInvPrev, 1.0f / float(cs.resourceSizePrev[0]), 1.0f / float(cs.resourceSizePrev[1]));
    set2(c.gRectSize, rectW, rectH);
    set2(c.gRectSizeInv, 1.0f / rectW, 1.0f / rectH);
    set2(c.gRectSizePrev, cs.rectSizePrev[0], cs.rectSizePrev[1]);
    set2(c.gResolutionScale, rectW / resW, rectH / resH);
    set2(c.gRectOffset, float(cs.rectOrigin[0]) / resW, float(cs.rectOrigin[1]) / resH);
    c.gPrintfAt[0] = cs.printfAt[0]; c.gPrintfAt[1] = cs.printfAt[1];
    c.gRectOrigin[0] = cs.rectOrigin[0]; c.gRectOrigin[1] = cs.rectOrigin[1];
    c.gRectSizeMinusOne[0] = cs.rectSize[0] - 1; c.gRectSizeMinusOne[1] = cs.rectSize[1] - 1;
    c.gTilesSizeMinusOne[0] = (cs.rectSize[0] + 15) / 16 - 1; c.gTilesSizeMinusOne[1] = (cs.rectSize[1] + 15) / 16 - 1;
    c.gOrthoMode = orthoMode;
    c.gUnproject = unproject;
    c.gDenoisingRange = cs.denoisingRange;
    c.gPlaneDistSensitivity = s.planeDistanceSensitivity;
    c.gStabilizationStrength = cs.accumulationMode == AccumulationMode::CONTINUE ? stabilizationStrength : 0.0f;
    c.gDebug = cs.debug;
    c.gSplitScreen = cs.splitScreen;
    c.gViewZScale = cs.viewZScale;
    c.gMinRectDimMulUnproject = std::min(rectW, rectH) * unproject;
    c.gFrameIndex = cs.frameIndex;
    c.gIsRectChanged = (cs.rectSize[0] != cs.rectSizePrev[0] || cs.rectSize[1] != cs.rectSizePrev[1]) ? 1 : 0;
}
} // namespace nrdb200
