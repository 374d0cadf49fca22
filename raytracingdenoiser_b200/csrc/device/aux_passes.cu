// Auxiliary passes on sm_90a: the split-screen passes of the three families (CommonSettings::splitScreen: the left part of the
// screen shows the noisy input) and the two passes of the REFERENCE denoiser.
// What has to be computed: Shaders/Include/REBLUR_SplitScreen.hlsli:11-47, RELAX_SplitScreen.hlsli:11-50, SIGMA_SplitScreen.hlsli:11-36,
// Shaders/Source/REFERENCE_TemporalAccumulation.cs.hlsl:19-30, REFERENCE_Copy.cs.hlsl:19-28.  All of them are pure streaming
// passes (one load, one store per texel, 128-bit accesses where the format allows).
#include "common.cuh"
#include "../constants.h"
#include "launch.h"

namespace nrdb200
{
namespace
{
constexpr float kFp16MaxAux = 65504.0f;

// ---- REBLUR / RELAX: out = in * (viewZ < denoisingRange) for uv.x <= splitScreen -------------------------------------------
struct SplitArgs
{
    Surf z, inDiff, inSpec, outDiff, outSpec;
    float rectSizeInvX, splitScreen, viewZScale, denoisingRange;
    int rectW, rectH;
    int hasDiff, hasSpec;
    int diffShift, specShift; // 1: checkerboarded input packed into the left half, pixel x shows column x >> 1 (REBLUR_SplitScreen.hlsli:24, :36; RELAX_SplitScreen.hlsli:24, :38)
    int rowBegin, rowEnd;
};
__global__ void __launch_bounds__(256) RadianceSplitScreenKernel(const __grid_constant__ SplitArgs a)
{
    const int x = blockIdx.x * 32 + threadIdx.x, y = a.rowBegin + blockIdx.y * 8 + threadIdx.y;
    if (x >= a.rectW || y >= a.rectH || y >= a.rowEnd) return;
    const float pixelUvX = __fmul_rn(__fadd_rn((float)x, 0.5f), a.rectSizeInvX);
    if (pixelUvX > a.splitScreen) return;
    const float viewZ = fabsf(LoadR32F(Near(a.z), x, y) * a.viewZScale);
    const bool keep = viewZ < a.denoisingRange;
    const uint2 zero = make_uint2(0u, 0u); // x * 0 in half precision: +0 (the sign of a negative input is not preserved; NaN inputs are not expected)
    if (a.hasDiff) *TexelPtrRW<uint2>(a.outDiff, x, y) = keep ? __ldg(TexelPtr<uint2>(Near(a.inDiff), x >> a.diffShift, y)) : zero;
    if (a.hasSpec) *TexelPtrRW<uint2>(a.outSpec, x, y) = keep ? __ldg(TexelPtr<uint2>(Near(a.inSpec), x >> a.specShift, y)) : zero;
}

// ---- SIGMA: out = (translucent ? IN_TRANSLUCENCY : IsLit(penumbra)) * (viewZ < denoisingRange) -------------------------------
struct SigmaSplitArgs
{
    Surf z, penumbra, translucency, out;
    float rectSizeInvX, splitScreen, viewZScale, denoisingRange;
    int rectW, rectH;
    int translucent;
    int rowBegin, rowEnd;
};
__global__ void __launch_bounds__(256) SigmaSplitScreenKernel(const __grid_constant__ SigmaSplitArgs a)
{
    const int x = blockIdx.x * 32 + threadIdx.x, y = a.rowBegin + blockIdx.y * 8 + threadIdx.y;
    if (x >= a.rectW || y >= a.rectH || y >= a.rowEnd) return;
    const float pixelUvX = __fmul_rn(__fadd_rn((float)x, 0.5f), a.rectSizeInvX);
    if (pixelUvX > a.splitScreen) return;
    const float viewZ = fabsf(LoadR32F(Near(a.z), x, y) * a.viewZScale);
    const bool keep = viewZ < a.denoisingRange;
    if (a.translucent)
        StoreU32(a.out, x, y, keep ? LoadU32(Near(a.translucency), x, y) : 0u); // RGBA8 -> float4 -> RGBA8 is the identity
    else
        StoreU8(a.out, x, y, keep && LoadR16F(Near(a.penumbra), x, y) >= kFp16MaxAux ? 255u : 0u);
}

// ---- REFERENCE -------------------------------------------------------------------------------------------------------------
struct ReferenceArgs
{
    Surf in, out;
    float accumSpeed, rectSizeInvX, splitScreen;
    int gridW, gridH;
    int rowBegin, rowEnd;
};
// history = lerp(history, input, accumSpeed) on the RGBA32F history (REFERENCE_TemporalAccumulation.cs.hlsl:24-29)
__global__ void __launch_bounds__(256) ReferenceAccumulateKernel(const __grid_constant__ ReferenceArgs a)
{
    const int x = blockIdx.x * 32 + threadIdx.x, y = a.rowBegin + blockIdx.y * 8 + threadIdx.y;
    if (x >= a.gridW || y >= a.gridH || y >= a.rowEnd || !Inside(a.out, x, y)) return;
    const f4 input = Inside(a.in, x, y) ? LoadRGBA16F(Near(a.in), x, y) : mk4(0.0f);
    float4* h = TexelPtrRW<float4>(a.out, x, y);
    const float4 history = *h;
    // lerp(a, b, t) = a + (b - a) * t, products and sums individually rounded like the oracle
    *h = make_float4(__fadd_rn(history.x, __fmul_rn(__fadd_rn(input.x, -history.x), a.accumSpeed)), __fadd_rn(history.y, __fmul_rn(__fadd_rn(input.y, -history.y), a.accumSpeed)),
                     __fadd_rn(history.z, __fmul_rn(__fadd_rn(input.z, -history.z), a.accumSpeed)), __fadd_rn(history.w, __fmul_rn(__fadd_rn(input.w, -history.w), a.accumSpeed)));
}
// OUT_SIGNAL = history for uv.x > splitScreen (REFERENCE_Copy.cs.hlsl:24-27)
__global__ void __launch_bounds__(256) ReferenceCopyKernel(const __grid_constant__ ReferenceArgs a)
{
    const int x = blockIdx.x * 32 + threadIdx.x, y = a.rowBegin + blockIdx.y * 8 + threadIdx.y;
    if (x >= a.gridW || y >= a.gridH || y >= a.rowEnd || !Inside(a.out, x, y)) return;
    const float pixelUvX = __fmul_rn(__fadd_rn((float)x, 0.5f), a.rectSizeInvX);
    if (!(pixelUvX > a.splitScreen)) return;
    const f4 v = Inside(a.in, x, y) ? LoadRGBA32F(Near(a.in), x, y) : mk4(0.0f);
    StoreRGBA16F(a.out, x, y, v);
}
} // namespace

cudaError_t LaunchAux(const PassLaunch& p)
{
    const int rows = p.rowEnd - p.rowBegin;
    const dim3 block(32, 8);
    const Family family = p.kind.family;
    Bindings b(p);
    if (family == Family::REBLUR || family == Family::RELAX) // split screen
    {
        SplitArgs a{};
        a.hasDiff = (p.kind.signals & SIGNAL_DIFFUSE) ? 1 : 0;
        a.hasSpec = (p.kind.signals & SIGNAL_SPECULAR) ? 1 : 0;
        unsigned diffCheckerboard, specCheckerboard;
        if (family == Family::REBLUR)
        {
            const ReblurConstants& c = *(const ReblurConstants*)p.constants;
            a.rectSizeInvX = c.gRectSizeInv[0]; a.splitScreen = c.gSplitScreen; a.viewZScale = c.gViewZScale; a.denoisingRange = c.gDenoisingRange;
            a.rectW = c.gRectSizeMinusOne[0] + 1; a.rectH = c.gRectSizeMinusOne[1] + 1;
            diffCheckerboard = c.gDiffCheckerboard; specCheckerboard = c.gSpecCheckerboard;
        }
        else
        {
            const RelaxConstants& c = *(const RelaxConstants*)p.constants;
            a.rectSizeInvX = c.gRectSizeInv[0]; a.splitScreen = c.gSplitScreen; a.viewZScale = c.gViewZScale; a.denoisingRange = c.gDenoisingRange;
            a.rectW = c.gRectSize[0]; a.rectH = c.gRectSize[1];
            diffCheckerboard = c.gDiffCheckerboard; specCheckerboard = c.gSpecCheckerboard;
        }
        a.diffShift = diffCheckerboard != 2 ? 1 : 0;
        a.specShift = specCheckerboard != 2 ? 1 : 0;
        a.z = b.Next();
        a.inDiff = b.Next(a.hasDiff);
        a.inSpec = b.Next(a.hasSpec);
        a.outDiff = b.Next(a.hasDiff);
        a.outSpec = b.Next(a.hasSpec);
        if (!b.Complete()) return cudaErrorInvalidValue;
        a.rowBegin = p.rowBegin; a.rowEnd = p.rowEnd;
        NRD_B200_LAUNCH(p, dim3((a.rectW + 31) / 32, (rows + 7) / 8), block, a, RadianceSplitScreenKernel);
        return cudaGetLastError();
    }
    if (family == Family::SIGMA) // split screen
    {
        const SigmaConstants& c = *(const SigmaConstants*)p.constants;
        SigmaSplitArgs a{};
        a.translucent = p.kind.translucent ? 1 : 0;
        a.rectSizeInvX = c.gRectSizeInv[0]; a.splitScreen = c.gSplitScreen; a.viewZScale = c.gViewZScale; a.denoisingRange = c.gDenoisingRange;
        a.rectW = c.gRectSizeMinusOne[0] + 1; a.rectH = c.gRectSizeMinusOne[1] + 1;
        a.z = b.Next(); a.penumbra = b.Next(); a.translucency = b.Next(a.translucent); a.out = b.Next();
        if (!b.Complete()) return cudaErrorInvalidValue;
        a.rowBegin = p.rowBegin; a.rowEnd = p.rowEnd;
        NRD_B200_LAUNCH(p, dim3((a.rectW + 31) / 32, (rows + 7) / 8), block, a, SigmaSplitScreenKernel);
        return cudaGetLastError();
    }
    if (family == Family::REFERENCE && (p.kind.pass == Pass::TemporalAccumulation || p.kind.pass == Pass::Copy))
    {
        ReferenceArgs a{};
        a.in = b.Next(); a.out = b.Next();
        if (!b.Complete()) return cudaErrorInvalidValue;
        a.gridW = p.gridW * 16; a.gridH = p.gridH * 16;
        a.rowBegin = p.rowBegin; a.rowEnd = p.rowEnd;
        const int w = p.preloadOnly ? 32 : a.out.w;
        if (p.kind.pass == Pass::Copy)
        {
            const ReferenceCopyConstants& c = *(const ReferenceCopyConstants*)p.constants;
            a.rectSizeInvX = c.gRectSizeInv[0]; a.splitScreen = c.gSplitScreen;
            NRD_B200_LAUNCH(p, dim3((w + 31) / 32, (rows + 7) / 8), block, a, ReferenceCopyKernel);
        }
        else
        {
            a.accumSpeed = ((const ReferenceAccumulateConstants*)p.constants)->gAccumSpeed;
            NRD_B200_LAUNCH(p, dim3((w + 31) / 32, (rows + 7) / 8), block, a, ReferenceAccumulateKernel);
        }
        return cudaGetLastError();
    }
    return cudaErrorNotSupported;
}

#if !defined(NRD_B200_NO_STRIPS)
cudaError_t SetPeerTableAux(int slot, const PeerTable* table, const cudaStream_t* stream) { return SetPeerTableThisTU(slot, table, stream); }
#endif
} // namespace nrdb200
