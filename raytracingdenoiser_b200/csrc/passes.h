// Pass identity: which kernel a pipeline runs.  The scheduler records one PassKind per pipeline when a recipe emits it and
// formats the shader file name from it (scheduler.cpp ShaderFileName); the executor and the launchers decide everything from
// the kind, never from the name.  Plain data without CUDA: the scheduler is compiled by the host compiler alone.
#pragma once
#include <stdint.h>

namespace nrdb200_abi
{
// "<family>[_Perf][_<signals>]_<pass>.cs".  Every pass name is the last part of its shader file name.
#define NRD_B200_PASSES(X)                                                                                                      \
    X(ClassifyTiles) X(SmoothTiles) X(HitDistReconstruction) X(HitDistReconstruction_5x5) X(PrePass) X(TemporalAccumulation)  \
    X(HistoryFix) X(HistoryClamping) X(Copy) X(AntiFirefly) X(AtrousSmem) X(Atrous) X(Blur) X(PostBlur)                        \
    X(PostBlur_NoTemporalStabilization) X(TemporalStabilization) X(SplitScreen) X(Validation) X(Float) X(Uint)

#define NRD_B200_PASS_ENUM(name) name,
enum class Pass : uint8_t { NRD_B200_PASSES(NRD_B200_PASS_ENUM) };
#undef NRD_B200_PASS_ENUM

// CLEAR: Clear_Float / Clear_Uint, the executor's own clears.  Validation (REBLUR, RELAX) has no kernel: its dispatch fails with
// Result::UNSUPPORTED.
enum class Family : uint8_t { CLEAR, REBLUR, RELAX, SIGMA, REFERENCE };

// PassKind::signals.  0 = a pipeline shared by every denoiser of its family (Clear_*, *_ClassifyTiles, SIGMA_SmoothTiles,
// SIGMA_Copy): the scheduler merges pipelines by shader file name, so a shared kind carries no signal and no translucency.
enum : uint8_t { SIGNAL_DIFFUSE = 1, SIGNAL_SPECULAR = 2, SIGNAL_SHADOW = 4 };

struct PassKind
{
    Family family;
    Pass pass;
    uint8_t signals = 0;      // SIGNAL_* bits
    bool perf = false;        // REBLUR_Perf_*: ReblurSettings::enablePerformanceMode
    bool translucent = false; // SIGMA_ShadowTranslucency_*: the shadow is a float4 in RGBA8 textures
};
} // namespace nrdb200_abi
