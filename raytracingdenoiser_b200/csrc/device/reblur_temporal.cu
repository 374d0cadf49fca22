// REBLUR temporal passes on sm_90a: TemporalAccumulation, HistoryFix, TemporalStabilization.
// Semantics: reference Shaders/Include/REBLUR_TemporalAccumulation.hlsli:11-931, REBLUR_HistoryFix.hlsli:11-463,
// REBLUR_TemporalStabilization.hlsli:11-367 with helpers from Common.hlsli / REBLUR_Common.hlsli (cited inline), default
// switches (CatRom on, STF on, SPECULAR_MOTION_V2, antilag mode 2), checkerboard OFF, no history-confidence /
// disocclusion-mix / base-colour inputs.  Reprojection footprints are selected with pinned arithmetic (common.cuh).
#include "reblur_math.cuh"
#include "launch.h"
#include "samplers.cuh"
#include "tma.cuh"

namespace nrdb200
{
using namespace rb;

// bilinear footprint: origin = floor(uv * size - 0.5), weights = frac   (pinned)
struct Bilinear
{
    float ox, oy, wx, wy;
};
__device__ __forceinline__ Bilinear GetBilinear(f2 uv, const float* size)
{
    float tx = __fadd_rn(__fmul_rn(uv.x, size[0]), -0.5f), ty = __fadd_rn(__fmul_rn(uv.y, size[1]), -0.5f);
    Bilinear b;
    b.ox = floorf(tx);
    b.oy = floorf(ty);
    b.wx = __fadd_rn(tx, -b.ox);
    b.wy = __fadd_rn(ty, -b.oy);
    return b;
}
__device__ __forceinline__ float ApplyBilinear(float s00, float s10, float s01, float s11, const Bilinear& f)
{
    return lerpf(lerpf(s00, s10, f.wx), lerpf(s01, s11, f.wx), f.wy);
}
__device__ __forceinline__ f4 CustomWeights(const Bilinear& f, f4 cw)
{
    float ox = 1.0f - f.wx, oy = 1.0f - f.wy;
    return mk4(cw.x * (ox * oy), cw.y * (f.wx * oy), cw.z * (ox * f.wy), cw.w * (f.wx * f.wy));
}
__device__ __forceinline__ float ApplyCustomWeights(float s00, float s10, float s01, float s11, f4 w)
{
    float sum = w.x + w.y + w.z + w.w;
    float r = s00 * w.x + s10 * w.y + s01 * w.z + s11 * w.w;
    return sum < 0.0001f ? 0.0f : r / sum;
}
__device__ __forceinline__ f4 InScreenBilinear(const Bilinear& f, const float* size) // Common.hlsli:287-295
{
    float x0 = (f.ox >= 0.0f && f.ox < size[0]) ? 1.0f : 0.0f, x1 = (f.ox + 1.0f >= 0.0f && f.ox + 1.0f < size[0]) ? 1.0f : 0.0f;
    float y0 = (f.oy >= 0.0f && f.oy < size[1]) ? 1.0f : 0.0f, y1 = (f.oy + 1.0f >= 0.0f && f.oy + 1.0f < size[1]) ? 1.0f : 0.0f;
    return mk4(x0 * y0, x1 * y0, x0 * y1, x1 * y1);
}

// thin-lens virtual position (Common.hlsli:404-461, NRD_USE_SPECULAR_MOTION_V2 = 1).  The kernel evaluates it for two hit
// distances: what does not depend on the hit distance is set up once per pixel (the compiler does not merge the two inlined
// copies of the dominant direction's powf).
struct XvirtualSetup
{
    f4 D;           // dominant direction, .w = dominant factor
    float magScale; // 1 / (1 + thin-lens term)
};
__device__ __forceinline__ XvirtualSetup SetupXvirtual(float curvature, float lengthX, f3 N, f3 V, float aLog)
{
    XvirtualSetup s;
    s.D = SpecularDominantDirectionLut(N, V, aLog); // aLog: roughness-table entry of the pixel's roughness
    float f = lengthX * (1.0f - fabsf(dot(N, V))) * fmaxf(curvature, 0.0f);
    s.magScale = 1.0f / (1.0f + f);
    return s;
}
__device__ __forceinline__ f3 GetXvirtual(const XvirtualSetup& s, float hitDist, float curvature, f3 X, f3 Xprev, f3 N, f3 V)
{
    f3 ray = xyz(s.D) * hitDist;
    f3 T, B;
    GetBasis(N, T, B);
    float Oz = -dot(N, ray);
    float Ox = dot(T, ray), Oy = dot(B, ray);
    float mag = 1.0f / (2.0f * curvature * Oz - 1.0f);
    mag *= s.magScale;
    float lenI = sqrtf(Ox * Ox + Oy * Oy + Oz * Oz) * fabsf(mag);
    f3 Iw = V * lenI;
    float closeness = saturate(length(Iw) / (hitDist + kEps));
    f3 origin = lerp3(Xprev, X, closeness * s.D.w);
    return origin - Iw * s.D.w;
}

__device__ __forceinline__ unsigned LoadPackedNrOrZero(const Surf& s, int x, int y) { return Inside(s, x, y) ? LoadU32(s, x, y) : 0u; }

// =============================================================================================
// Temporal accumulation
// =============================================================================================
struct TaArgs
{
    ReblurConstants c;
    Surf tiles, nr, z, mv, prevZ, prevNr, prevInternal;
    Surf mix, diffConfidence, specConfidence; // optional R8_UNORM inputs (REBLUR_TemporalAccumulation.hlsli:220-221, :327-328, :830-831), read only when the constants say so
    Surf inDiff, inSpec, histDiff, histSpec, histDiffFast, histSpecFast, prevHitDist, inHitDist;
    Surf outDiff, outSpec, outDiffFast, outSpecFast, outHitDist, outData1, outData2;
    Surf guide;          // decoded guides of the current frame (surf.h PassLaunch::guide)
    const float4* lut;   // roughness table (surf.h PassLaunch::roughnessLut)
    int rowBegin, rowEnd;
    int perf;            // REBLUR_PERFORMANCE_MODE: no CatRom history filters (REBLUR_Config.hlsli:196-202)
};

// GENERAL = false: the kernel of the default configuration, the only one compiled with these switches as constants --
// perspective projection, 2.5D screen-space motion vectors, no checkerboard, no history-confidence / disocclusion-mix inputs,
// specular pre-pass on, performance mode off.  GENERAL = true reads them from the constants (LaunchTa picks).
template <bool DIFF, bool SPEC, bool GENERAL = false>
#ifndef NRD_B200_TA_MIN_BLOCKS
#define NRD_B200_TA_MIN_BLOCKS 5 // <= 96 registers: 5 x 128 threads per SM instead of 3 (measured 1.7x on this kernel)
#endif
__global__ void __launch_bounds__(128, NRD_B200_TA_MIN_BLOCKS) ReblurTemporalAccumulationKernel(const __grid_constant__ TaArgs a)
{
    const ReblurConstants& c = a.c;
    const float orthoMode = GENERAL ? c.gOrthoMode : 0.0f;
    const bool worldSpaceMv = GENERAL && c.gMvScale[3] != 0.0f;
    const bool hasConfidence = GENERAL && c.gHasHistoryConfidence;
    const bool hasThresholdMix = GENERAL && c.gHasDisocclusionThresholdMix;
    const bool specPrepass = !GENERAL || c.gSpecPrepassBlurRadius != 0.0f;
    const bool perf = GENERAL && a.perf;
    const int x = blockIdx.x * 32 + threadIdx.x;
    const int y = a.rowBegin + blockIdx.y * 4 + threadIdx.y;
    const int maxX = c.gRectSizeMinusOne[0], maxY = c.gRectSizeMinusOne[1];
    if (x > maxX || y > maxY || y >= a.rowEnd) return;
    if (LoadU8(Near(a.tiles), x >> 4, y >> 4) != 0) return;
    const float viewZ = fabsf(LoadR32F(Near(a.z), x, y) * c.gViewZScale);
    if (viewZ > c.gDenoisingRange) return;

    const f2 pixelUv = PixelUv(x, y, c.gRectSizeInv);
    const f3 Xv = ReconstructViewPosition(pixelUv, c.gFrustum, viewZ, orthoMode);
    const f3 X = PinnedRotate(c.gViewToWorld, Xv);
    const unsigned checkerboard = GENERAL ? CheckerBoard(x, y, c.gFrameIndex) : 0u;

    // 3x3 neighbourhood: averaged normal (2x2 corner), roughness moments, min hit distance for tracking
    f3 Navg = mk3(0.0f);
    f3 n10 = mk3(0.0f), n01 = mk3(0.0f);
    float hitDistForTracking = kInf, roughnessM1 = 0.0f, roughnessM2 = 0.0f;
#pragma unroll
    for (int j = 0; j <= 2; j++)
#pragma unroll
        for (int i = 0; i <= 2; i++)
        {
            int px = clampi(x + i - 1, 0, maxX), py = clampi(y + j - 1, 0, maxY);
            const Guide g = LoadGuide(Near(a.guide), Near(a.nr), px, py);
            if (i < 2 && j < 2) Navg = Navg + g.N;
            if (i == 2 && j == 1) n10 = g.N;
            if (i == 1 && j == 2) n01 = g.N;
            if (SPEC)
            {
                float h = !specPrepass ? LoadRGBA16F(Near(a.inSpec), px, py).w : LoadR16F(Near(a.inHitDist), px, py);
                hitDistForTracking = fminf(hitDistForTracking, h == 0.0f ? kInf : h);
                float r2 = g.roughness * g.roughness;
                roughnessM1 += r2;
                roughnessM2 += r2 * r2;
            }
        }
    Navg = Navg * 0.25f;

    const Guide g0 = LoadGuideLut(Near(a.guide), Near(a.nr), a.lut, x, y);
    const f3 N = g0.N;
    const float roughness = g0.roughness, materialID = g0.materialID;

    float roughnessModified = 0.0f, roughnessSigma = 0.0f, hitDistNormalization = 0.0f;
    RngHash rng;
    if (SPEC)
    {
        roughnessModified = ModifiedRoughness(roughness, Navg);
        roughnessM1 *= 1.0f / 9.0f;
        roughnessM2 *= 1.0f / 9.0f;
        roughnessSigma = GetStdDev(roughnessM1, roughnessM2);
        rng.Initialize(x, y, c.gFrameIndex);
        hitDistForTracking = hitDistForTracking == kInf ? 0.0f : hitDistForTracking;
        hitDistNormalization = (c.gHitDistParams[0] + viewZ * c.gHitDistParams[1]) * g0.hitK;
        hitDistForTracking *= !specPrepass ? hitDistNormalization : 1.0f;
        StoreR16F(a.outHitDist, x, y, hitDistForTracking);
    }

    // previous position and surface-motion uv
    const f4 mvRaw = LoadRGBA16F(Near(a.mv), x, y);
    f3 mv = mk3(__fmul_rn(mvRaw.x, c.gMvScale[0]), __fmul_rn(mvRaw.y, c.gMvScale[1]), __fmul_rn(mvRaw.z, c.gMvScale[2]));
    f3 Xprev = X;
    f2 smbPixelUv = mk2(__fadd_rn(pixelUv.x, mv.x), __fadd_rn(pixelUv.y, mv.y));
    const f3 camDelta = mk3(c.gCameraDelta[0], c.gCameraDelta[1], c.gCameraDelta[2]);
    if (!worldSpaceMv)
    {
        if (c.gMvScale[2] == 0.0f) mv.z = __fadd_rn(PinnedRow(c.gWorldToViewPrev, 2, X.x, X.y, X.z), -viewZ);
        float viewZprev = __fadd_rn(viewZ, mv.z);
        f3 Xvprevlocal = ReconstructViewPosition(smbPixelUv, c.gFrustumPrev, viewZprev, orthoMode);
        f3 r = PinnedRotateInverse(c.gWorldToViewPrev, Xvprevlocal);
        Xprev = mk3(__fadd_rn(r.x, camDelta.x), __fadd_rn(r.y, camDelta.y), __fadd_rn(r.z, camDelta.z));
    }
    else
    {
        Xprev = mk3(__fadd_rn(X.x, mv.x), __fadd_rn(X.y, mv.y), __fadd_rn(X.z, mv.z));
        smbPixelUv = GetScreenUv(c.gWorldToClipPrev, Xprev);
    }

    // previous viewZ / internal data in the 4x4 CatRom footprint (12 texels, corners unused) around the bilinear origin b.
    // A texel is occluded when its plane distance exceeds the threshold of its quadrant, and the thresholds need the previous
    // normal of the inner 2x2 first.  The 8 outer texels only decide whether all 12 pass (CatRom allowed), so they are reduced as
    // they are loaded: per quadrant the largest plane distance, plus one flag that is cleared by a material mismatch or a NaN
    // distance (NaN fails `d <= thr`, fmaxf would drop it).  `max <= thr` is then exactly `d <= thr` for both texels.
    const Bilinear smbF = GetBilinear(smbPixelUv, c.gRectSizePrev);
    const int bx = (int)smbF.ox, by = (int)smbF.oy;
    const int W1 = a.prevZ.w - 1, H1 = a.prevZ.h - 1;
    const float XvprevZ = PinnedRow(c.gWorldToViewPrev, 2, Xprev.x, Xprev.y, Xprev.z);
    const float minMaterial = fminf(c.gSpecMinMaterial, c.gDiffMinMaterial);
    const float centerMat = fmaxf(materialID, minMaterial);
    // inner 2x2, index [row * 2 + col] <-> texel (bx + col, by + row), i.e. gather order 00, 10, 01, 11
    float pz[4];
    unsigned pid[4];
    float outerDist[4] = {0.0f, 0.0f, 0.0f, 0.0f}; // per quadrant, same order
    bool outerPass = true;
    // prevZ and prevInternal are full-resolution pool surfaces of one geometry: one row lookup serves both
#pragma unroll
    for (int r = 0; r < 4; r++)
    {
        const RowRef row = RefRow(a.prevZ, clampi(by - 1 + r, 0, H1));
#pragma unroll
        for (int q = 0; q < 4; q++)
        {
            if ((r == 0 || r == 3) && (q == 0 || q == 3)) continue;
            const int tx = clampi(bx - 1 + q, 0, W1);
            const float z = fabsf(__ldg(TexelAt<float>(a.prevZ, row, tx)) * c.gViewZScale);
            const unsigned id = __ldg(TexelAt<unsigned short>(a.prevInternal, row, tx));
            if (r >= 1 && r <= 2 && q >= 1 && q <= 2)
            {
                pz[(r - 1) * 2 + q - 1] = z;
                pid[(r - 1) * 2 + q - 1] = id;
            }
            else
            {
                const float d = fabsf(z - XvprevZ);
                const int k = (r < 2 ? 0 : 2) + (q < 2 ? 0 : 1);
                outerDist[k] = fmaxf(outerDist[k], d);
                outerPass &= d == d && centerMat == fmaxf(UnpackInternalData(id).z, minMaterial);
            }
        }
    }

    // previous normal averaged over the valid part of the 2x2 footprint
    f3 smbNavg;
    {
        int px = (int)fmaxf(smbF.ox, 0.0f), py = (int)fmaxf(smbF.oy, 0.0f); // uint2(origin): float -> uint saturates at 0
        float w00 = pz[0] < c.gDenoisingRange ? 1.0f : 0.0f, w10 = pz[1] < c.gDenoisingRange ? 1.0f : 0.0f;
        float w01 = pz[2] < c.gDenoisingRange ? 1.0f : 0.0f, w11 = pz[3] < c.gDenoisingRange ? 1.0f : 0.0f;
        auto sumN = [&](const Surf& prevNr) {
            f3 t = DecodeGuide(LoadPackedNrOrZero(prevNr, px, py)).N * w00;
            t = t + DecodeGuide(LoadPackedNrOrZero(prevNr, px + 1, py)).N * w10;
            t = t + DecodeGuide(LoadPackedNrOrZero(prevNr, px, py + 1)).N * w01;
            return t + DecodeGuide(LoadPackedNrOrZero(prevNr, px + 1, py + 1)).N * w11;
        };
        f3 s = FootprintLocal(a.prevNr, py, py + 1) ? sumN(Near(a.prevNr)) : sumN(a.prevNr);
        float sum = w00 + w10 + w01 + w11;
        smbNavg = Rotate(c.gWorldPrevToWorld, s * (1.0f / (sum == 0.0f ? 1.0f : sum)));
    }

    // parallax in pixels (both definitions, Common.hlsli:319-332)
    const f2 rectSize = mk2(c.gRectSize[0], c.gRectSize[1]);
    const f2 uvPrevOfXprevPlusDelta = GetScreenUv(c.gWorldToClipPrev, Xprev + camDelta);
    f2 d1 = (uvPrevOfXprevPlusDelta - (orthoMode == 0.0f ? smbPixelUv : pixelUv)) * rectSize;
    f2 d2 = (GetScreenUv(c.gWorldToClip, Xprev - camDelta) - (orthoMode == 0.0f ? pixelUv : smbPixelUv)) * rectSize;
    const float smbParallaxInPixels1 = length(d1), smbParallaxInPixels2 = length(d2);
    const float smbParallaxInPixelsMax = fmaxf(smbParallaxInPixels1, smbParallaxInPixels2);
    const float smbParallaxInPixelsMin = fminf(smbParallaxInPixels1, smbParallaxInPixels2);

    // disocclusion threshold
    const float pixelSize = c.gUnproject * lerpf(viewZ, 1.0f, fabsf(orthoMode));
    const float frustumSize = c.gMinRectDimMulUnproject * lerpf(viewZ, 1.0f, fabsf(orthoMode));
    float disocclusionThresholdMix = 0.0f;
    if (materialID == c.gStrandMaterialID) disocclusionThresholdMix = pixelSize / (pixelSize + c.gStrandThickness);
    if (hasThresholdMix) disocclusionThresholdMix = LoadR8Unorm(Near(a.mix), x, y);
    float disocclusionThreshold = lerpf(c.gDisocclusionThreshold, c.gDisocclusionThresholdAlternate, disocclusionThresholdMix);
    const float smallParallax = LinearStep(0.25f, 0.0f, smbParallaxInPixelsMax);
    disocclusionThreshold += 0.05f * smallParallax;

    const f3 V = orthoMode == 0.0f ? normalize(-X) : mk3(c.gViewVectorWorld[0], c.gViewVectorWorld[1], c.gViewVectorWorld[2]);
    const float NoV = fabsf(dot(N, V));
    const float NoVstrict = lerpf(NoV, 1.0f, saturate(smbParallaxInPixelsMax / 30.0f));
    const float almostZeroAngle = 0.0174524064f; // cos(89 deg)
    float thrBase = frustumSize * saturate(disocclusionThreshold / fmaxf(0.01f, NoVstrict));
    thrBase *= dot(smbNavg, Navg) > almostZeroAngle - 0.25f * smallParallax ? 1.0f : 0.0f;
    const f4 inScreen = InScreenBilinear(smbF, c.gRectSizePrev);
    const f4 smbThr = mk4(thrBase * inScreen.x - kEps, thrBase * inScreen.y - kEps, thrBase * inScreen.z - kEps, thrBase * inScreen.w - kEps);

    // occlusion of the inner texels: plane distance against the quadrant's threshold, then material ID
    auto innerOcclusion = [&](int k, float thr) {
        float o = fabsf(pz[k] - XvprevZ) <= thr ? 1.0f : 0.0f;
        return o * (centerMat == fmaxf(UnpackInternalData(pid[k]).z, minMaterial) ? 1.0f : 0.0f);
    };
    const f4 smbOcclusion = mk4(innerOcclusion(0, smbThr.x), innerOcclusion(1, smbThr.y), innerOcclusion(2, smbThr.z), innerOcclusion(3, smbThr.w));
    const f4 smbOcclusionWeights = CustomWeights(smbF, smbOcclusion);
    const bool outerAll = outerPass && outerDist[0] <= smbThr.x && outerDist[1] <= smbThr.y && outerDist[2] <= smbThr.z && outerDist[3] <= smbThr.w;
    const bool smbAllowCatRom = smbOcclusion.x + smbOcclusion.y + smbOcclusion.z + smbOcclusion.w > 3.5f && outerAll && !perf;
    float fbits = smbOcclusion.x + smbOcclusion.y * 2.0f + smbOcclusion.z * 4.0f + smbOcclusion.w * 8.0f;

    const f3 id00 = UnpackInternalData(pid[0]), id10 = UnpackInternalData(pid[1]), id01 = UnpackInternalData(pid[2]), id11 = UnpackInternalData(pid[3]);
    float diffAccumSpeed = ApplyCustomWeights(id00.x, id10.x, id01.x, id11.x, smbOcclusionWeights);
    float smbSpecAccumSpeed = ApplyCustomWeights(id00.y, id10.y, id01.y, id11.y, smbOcclusionWeights);

    // footprint quality
    const f3 smbVprev = orthoMode == 0.0f ? normalize(camDelta - Xprev) : mk3(c.gViewVectorWorldPrev[0], c.gViewVectorWorldPrev[1], c.gViewVectorWorldPrev[2]);
    const float NoVprev = fabsf(dot(N, smbVprev));
    float sizeQuality = (NoVprev + 1e-3f) / (NoV + 1e-3f);
    sizeQuality *= sizeQuality;
    sizeQuality = lerpf(0.1f, 1.0f, saturate(sizeQuality));
    float smbFootprintQuality = Sqrt01(ApplyBilinear(smbOcclusion.x, smbOcclusion.y, smbOcclusion.z, smbOcclusion.w, smbF)) * sizeQuality;

    const f2 smbSamplePos = mk2(saturate(smbPixelUv.x) * c.gRectSizePrev[0], saturate(smbPixelUv.y) * c.gRectSizePrev[1]);

    float specAccumSpeed = 0.0f, curvature = 0.0f, virtualHistoryAmount = 0.0f;
    if (SPEC)
    {
        float specHistoryConfidence = smbFootprintQuality;
        if (hasConfidence) specHistoryConfidence *= LoadR8Unorm(Near(a.specConfidence), x, y);
        smbSpecAccumSpeed *= lerpf(specHistoryConfidence, 1.0f, 1.0f / (1.0f + smbSpecAccumSpeed));
        smbSpecAccumSpeed = fminf(smbSpecAccumSpeed, c.gMaxAccumulatedFrameNum);
        const f4 spec = LoadRGBA16F(Near(a.inSpec), x, y);

        // curvature along the predicted motion (REBLUR_TemporalAccumulation.hlsli:364-447)
        {
            f2 uvForZeroParallax = orthoMode == 0.0f ? smbPixelUv : pixelUv;
            f2 deltaUv = (uvForZeroParallax - uvPrevOfXprevPlusDelta) * rectSize;
            float invP = 1.0f / fmaxf(smbParallaxInPixels1, 1.0f / 256.0f);
            deltaUv = deltaUv * invP;

            f3 x10, x01;
            {
                f2 uv = mk2(pixelUv.x + c.gRectSizeInv[0], pixelUv.y);
                f3 xw = Rotate(c.gViewToWorld, ReconstructViewPosition(uv, c.gFrustum, 1.0f, orthoMode));
                f3 v = orthoMode == 0.0f ? normalize(-xw) : mk3(c.gViewVectorWorld[0], c.gViewVectorWorld[1], c.gViewVectorWorld[2]);
                f3 o = orthoMode == 0.0f ? mk3(0.0f) : xw;
                x10 = o + v * (dot(X - o, N) / dot(N, v));
            }
            {
                f2 uv = mk2(pixelUv.x, pixelUv.y + c.gRectSizeInv[1]);
                f3 xw = Rotate(c.gViewToWorld, ReconstructViewPosition(uv, c.gFrustum, 1.0f, orthoMode));
                f3 v = orthoMode == 0.0f ? normalize(-xw) : mk3(c.gViewVectorWorld[0], c.gViewVectorWorld[1], c.gViewVectorWorld[2]);
                f3 o = orthoMode == 0.0f ? mk3(0.0f) : xw;
                x01 = o + v * (dot(X - o, N) / dot(N, v));
            }
            f2 w = mk2(fabsf(deltaUv.x) + 1.0f / 256.0f, fabsf(deltaUv.y) + 1.0f / 256.0f);
            float ws = 1.0f / (w.x + w.y);
            w = w * ws;
            f3 xm = x10 * w.x + x01 * w.y;
            f3 n = normalize(n10 * w.x + n01 * w.y);

            // high parallax: replace the 1-pixel edge by a longer one along the motion
            float deltaUvLenFixed = smbParallaxInPixelsMin;
            deltaUvLenFixed *= 1.0f + c.gFramerateScale * Bayer4x4(x, y, c.gFrameIndex);
            // pinned: the snapped uv selects a texel
            float mu = __fadd_rn(pixelUv.x, __fmul_rn(__fmul_rn(deltaUvLenFixed, deltaUv.x), c.gRectSizeInv[0]));
            float mvv = __fadd_rn(pixelUv.y, __fmul_rn(__fmul_rn(deltaUvLenFixed, deltaUv.y), c.gRectSizeInv[1]));
            float fx = floorf(__fmul_rn(mu, c.gRectSize[0])), fy = floorf(__fmul_rn(mvv, c.gRectSize[1]));
            int ix = (int)fx, iy = (int)fy;
            if (deltaUvLenFixed > 1.0f && (unsigned)ix <= (unsigned)maxX && (unsigned)iy <= (unsigned)maxY)
            {
                f2 motionUvHigh = mk2(__fmul_rn(__fadd_rn(fx, 0.5f), c.gRectSizeInv[0]), __fmul_rn(__fadd_rn(fy, 0.5f), c.gRectSizeInv[1]));
                const bool tapLocal = RowsLocal(a.z, iy, iy);
                float zHigh = fabsf((tapLocal ? LoadR32F(Near(a.z), ix, iy) : LoadR32F(a.z, ix, iy)) * c.gViewZScale);
                f3 xHigh = Rotate(c.gViewToWorld, ReconstructViewPosition(motionUvHigh, c.gFrustum, zHigh, orthoMode));
                f3 nHigh = DecodeGuide(tapLocal ? LoadU32(Near(a.nr), ix, iy) : LoadU32(a.nr, ix, iy)).N;
                float zError = fabsf(zHigh - viewZ) / fmaxf(zHigh, viewZ);
                if (zError < 0.1f)
                {
                    n = nHigh;
                    xm = xHigh;
                }
            }
            f3 edge = xm - X;
            curvature = dot(n - N, edge) * PositiveRcp(dot(edge, edge));
        }

        // virtual motion
        const float lengthX = length(X);
        const XvirtualSetup xs = SetupXvirtual(curvature, lengthX, N, V, g0.aLog);
        const f3 Xvirtual = GetXvirtual(xs, hitDistForTracking, curvature, X, Xprev, N, V);
        const float XvirtualLength = length(Xvirtual);
        f2 vmbPixelUv = GetScreenUv(c.gWorldToClipPrev, Xvirtual);
        if (materialID == c.gCameraAttachedReflectionMaterialID) vmbPixelUv = smbPixelUv;
        f2 vmbDelta = vmbPixelUv - smbPixelUv;
        const float vmbPixelsTraveled = length(vmbDelta * rectSize);

        const Bilinear vmbF = GetBilinear(vmbPixelUv, c.gRectSizePrev);
        const int vx = (int)vmbF.ox, vy = (int)vmbF.oy;
        // 2x2 footprint fetches (clamped, like Gather with a clamp sampler)
        const int vx0 = clampi(vx, 0, W1), vx1 = clampi(vx + 1, 0, W1), vy0 = clampi(vy, 0, H1), vy1 = clampi(vy + 1, 0, H1);
        f2 rrp = RelaxedRoughnessWeightParams(roughness * roughness, c.gRoughnessFraction, 0.003f);
        unsigned vmbNr[4];
        float vmbZ[4];
        unsigned vmbId[4];
        {
            // prevNr, prevZ and prevInternal are full-resolution pool surfaces of one geometry: one lookup per row serves all three
            const RowRef r0 = RefRow(a.prevNr, vy0), r1 = RefRow(a.prevNr, vy1);
            vmbNr[0] = __ldg(TexelAt<unsigned>(a.prevNr, r0, vx0)); vmbNr[1] = __ldg(TexelAt<unsigned>(a.prevNr, r0, vx1));
            vmbNr[2] = __ldg(TexelAt<unsigned>(a.prevNr, r1, vx0)); vmbNr[3] = __ldg(TexelAt<unsigned>(a.prevNr, r1, vx1));
            vmbZ[0] = __ldg(TexelAt<float>(a.prevZ, r0, vx0)); vmbZ[1] = __ldg(TexelAt<float>(a.prevZ, r0, vx1));
            vmbZ[2] = __ldg(TexelAt<float>(a.prevZ, r1, vx0)); vmbZ[3] = __ldg(TexelAt<float>(a.prevZ, r1, vx1));
            vmbId[0] = __ldg(TexelAt<unsigned short>(a.prevInternal, r0, vx0)); vmbId[1] = __ldg(TexelAt<unsigned short>(a.prevInternal, r0, vx1));
            vmbId[2] = __ldg(TexelAt<unsigned short>(a.prevInternal, r1, vx0)); vmbId[3] = __ldg(TexelAt<unsigned short>(a.prevInternal, r1, vx1));
        }
        f4 vmbRoughness = mk4(DecodeGuide(vmbNr[0]).roughness, DecodeGuide(vmbNr[1]).roughness, DecodeGuide(vmbNr[2]).roughness, DecodeGuide(vmbNr[3]).roughness);
        const float jf = SmoothStep(1.0f, 0.0f, smbParallaxInPixelsMax);
        f4 roughnessWeight;
        roughnessWeight.x = lerpf(jf, 1.0f, NonExpWeightWithSigma(vmbRoughness.x * vmbRoughness.x, rrp.x, rrp.y, roughnessSigma));
        roughnessWeight.y = lerpf(jf, 1.0f, NonExpWeightWithSigma(vmbRoughness.y * vmbRoughness.y, rrp.x, rrp.y, roughnessSigma));
        roughnessWeight.z = lerpf(jf, 1.0f, NonExpWeightWithSigma(vmbRoughness.z * vmbRoughness.z, rrp.x, rrp.y, roughnessSigma));
        roughnessWeight.w = lerpf(jf, 1.0f, NonExpWeightWithSigma(vmbRoughness.w * vmbRoughness.w, rrp.x, rrp.y, roughnessSigma));
        float virtualHistoryRoughnessBasedConfidence = ApplyBilinear(roughnessWeight.x, roughnessWeight.y, roughnessWeight.z, roughnessWeight.w, vmbF);

        // stochastic bilinear pick of the previous normal (STF): one of the 4 footprint texels, point sampled with clamp
        auto stochasticNr = [&](f2 uv) {
            Bilinear f = GetBilinear(uv, c.gRectSizePrev);
            float r0 = rng.GetFloat(), r1 = rng.GetFloat();
            float ox = f.ox + (f.wx >= r0 ? 1.0f : 0.0f), oy = f.oy + (f.wy >= r1 ? 1.0f : 0.0f);
            // (origin + 0.5) / size * resolutionScale -> nearest texel = origin, clamped to the texture
            int tx = (int)floorf((ox + 0.5f) / c.gRectSizePrev[0] * c.gResolutionScalePrev[0] * (float)a.prevNr.w);
            int ty = (int)floorf((oy + 0.5f) / c.gRectSizePrev[1] * c.gResolutionScalePrev[1] * (float)a.prevNr.h);
            return DecodeGuide(LoadU32(a.prevNr, clampi(tx, 0, W1), clampi(ty, 0, H1)));
        };
        const Guide vmbGuide = stochasticNr(vmbPixelUv);
        const f3 vmbN = Rotate(c.gWorldPrevToWorld, vmbGuide.N);
        const float Dfactor = xs.D.w;
        float virtualHistoryNormalBasedConfidence = 1.0f / (1.0f + 0.5f * Dfactor * saturate(length(N - vmbN) - kNormalEncodingError) * vmbPixelsTraveled);

        if (smbFootprintQuality == 0.0f) smbNavg = vmbN;

        // virtual-motion disocclusion: plane distance, roughness, material
        f4 vmbOcclusion;
        {
            float thr = disocclusionThreshold * frustumSize * lerpf(0.25f, 1.0f, NoV);
            thr *= dot(vmbN, N) > almostZeroAngle ? 1.0f : 0.0f;
            thr *= dot(vmbN, smbNavg) > almostZeroAngle ? 1.0f : 0.0f;
            f4 inS = InScreenBilinear(vmbF, c.gRectSizePrev);
            f4 vmbThr = mk4(thr * inS.x - kEps, thr * inS.y - kEps, thr * inS.z - kEps, thr * inS.w - kEps);
            f4 vmbViewZ = mk4(fabsf(vmbZ[0] * c.gViewZScale), fabsf(vmbZ[1] * c.gViewZScale), fabsf(vmbZ[2] * c.gViewZScale), fabsf(vmbZ[3] * c.gViewZScale));
            f3 vmbVv = ReconstructViewPosition(vmbPixelUv, c.gFrustumPrev, 1.0f, 0.0f);
            f3 vmbV = RotateInverse(c.gWorldToViewPrev, vmbVv);
            float NoXcurr = dot(N, Xprev - camDelta);
            float nxy = N.x * vmbV.x + N.y * vmbV.y, nz = N.z * vmbV.z;
            auto planeDist = [&](float z) { return fabsf(nxy * (orthoMode == 0.0f ? z : orthoMode) + nz * z - NoXcurr); };
            vmbOcclusion.x = (planeDist(vmbViewZ.x) <= vmbThr.x ? 1.0f : 0.0f) * (roughnessWeight.x >= 0.5f ? 1.0f : 0.0f);
            vmbOcclusion.y = (planeDist(vmbViewZ.y) <= vmbThr.y ? 1.0f : 0.0f) * (roughnessWeight.y >= 0.5f ? 1.0f : 0.0f);
            vmbOcclusion.z = (planeDist(vmbViewZ.z) <= vmbThr.z ? 1.0f : 0.0f) * (roughnessWeight.z >= 0.5f ? 1.0f : 0.0f);
            vmbOcclusion.w = (planeDist(vmbViewZ.w) <= vmbThr.w ? 1.0f : 0.0f) * (roughnessWeight.w >= 0.5f ? 1.0f : 0.0f);
        }
        const f3 v00 = UnpackInternalData(vmbId[0]), v10 = UnpackInternalData(vmbId[1]);
        const f3 v01 = UnpackInternalData(vmbId[2]), v11 = UnpackInternalData(vmbId[3]);
        {
            float cm = fmaxf(materialID, c.gSpecMinMaterial);
            vmbOcclusion.x *= cm == fmaxf(v00.z, c.gSpecMinMaterial) ? 1.0f : 0.0f;
            vmbOcclusion.y *= cm == fmaxf(v10.z, c.gSpecMinMaterial) ? 1.0f : 0.0f;
            vmbOcclusion.z *= cm == fmaxf(v01.z, c.gSpecMinMaterial) ? 1.0f : 0.0f;
            vmbOcclusion.w *= cm == fmaxf(v11.z, c.gSpecMinMaterial) ? 1.0f : 0.0f;
        }
        fbits += vmbOcclusion.x * 16.0f + vmbOcclusion.y * 32.0f + vmbOcclusion.z * 64.0f + vmbOcclusion.w * 128.0f;

        const f4 vmbOcclusionWeights = CustomWeights(vmbF, vmbOcclusion);
        float vmbSpecAccumSpeed = ApplyCustomWeights(v00.y, v10.y, v01.y, v11.y, vmbOcclusionWeights);
        float vmbFootprintQuality = Sqrt01(ApplyBilinear(vmbOcclusion.x, vmbOcclusion.y, vmbOcclusion.z, vmbOcclusion.w, vmbF));
        vmbSpecAccumSpeed *= lerpf(vmbFootprintQuality, 1.0f, 1.0f / (1.0f + vmbSpecAccumSpeed));
        const bool vmbAllowCatRom = (vmbOcclusion.x + vmbOcclusion.y + vmbOcclusion.z + vmbOcclusion.w > 3.5f) && smbAllowCatRom; // (smbAllowCatRom is false in performance mode)

        // how far (in angle) the virtual motion may have travelled
        float curvatureAngleTan = pixelSize * fabsf(curvature) * fmaxf(vmbPixelsTraveled / fmaxf(NoV, 0.01f), 1.0f) * 2.0f;
        const float curvatureAngle = atanf(curvatureAngleTan);
        const float lobeTanHalfAngle = LobeTanHalfAngle(roughnessModified, kLobeVolume / (1.0f + vmbSpecAccumSpeed));
        const float lobeHalfAngle = fmaxf(atanf(lobeTanHalfAngle), kNormalEncodingError);
        float normalWeight = EncodingAwareNormalWeight(N, vmbN, lobeHalfAngle, curvatureAngle, kNormalEncodingError);
        normalWeight = lerpf(SmoothStep(1.0f, 0.0f, vmbPixelsTraveled), 1.0f, normalWeight);
        virtualHistoryNormalBasedConfidence = fminf(virtualHistoryNormalBasedConfidence, normalWeight);

        virtualHistoryAmount = SmoothStep(0.05f, 0.95f, Dfactor) * virtualHistoryNormalBasedConfidence;

        // virtual parallax difference against the previous frame's hit distance
        float virtualHistoryParallaxBasedConfidence;
        {
            float hitDistForTrackingPrev = SampleLinear1(a.prevHitDist, vmbPixelUv.x * c.gResolutionScalePrev[0], vmbPixelUv.y * c.gResolutionScalePrev[1]);
            f3 XvirtualPrev = GetXvirtual(xs, hitDistForTrackingPrev, curvature, X, Xprev, N, V);
            f2 vmbPixelUvPrev = GetScreenUv(c.gWorldToClipPrev, XvirtualPrev);
            if (materialID == c.gCameraAttachedReflectionMaterialID) vmbPixelUvPrev = smbPixelUv;
            float pixelSizeAtXvirtual = c.gUnproject * lerpf(XvirtualLength, 1.0f, fabsf(orthoMode));
            float r = (lobeTanHalfAngle + curvatureAngle) * fminf(hitDistForTracking, hitDistForTrackingPrev) / pixelSizeAtXvirtual;
            float d = length((vmbPixelUvPrev - vmbPixelUv) * rectSize);
            r = fmaxf(r, 0.1f);
            virtualHistoryParallaxBasedConfidence = LinearStep(r, 0.0f, d);
        }

        // prev-prev normal & roughness test, one tap further along the virtual motion
        {
            float stepBetweenTaps = fminf(vmbPixelsTraveled * c.gFramerateScale, 2.0f) + vmbPixelsTraveled;
            float invLen = rsqrtf(dot(vmbDelta, vmbDelta));
            f2 dir = mk2(vmbDelta.x * invLen / c.gRectSizePrev[0], vmbDelta.y * invLen / c.gRectSizePrev[1]);
            f2 rrp2 = RelaxedRoughnessWeightParams(vmbGuide.roughness * vmbGuide.roughness, c.gRoughnessFraction, 0.003f);
            f2 uvPrev = mk2(vmbPixelUv.x + dir.x * stepBetweenTaps, vmbPixelUv.y + dir.y * stepBetweenTaps);
            Guide gp = stochasticNr(uvPrev);
            float wn = EncodingAwareNormalWeight(vmbGuide.N, gp.N, lobeHalfAngle, curvatureAngle * (1.0f + stepBetweenTaps), kNormalEncodingError);
            float wr = NonExpWeightWithSigma(gp.roughness * gp.roughness, rrp2.x, rrp2.y, roughnessSigma);
            float k = saturate(stepBetweenTaps);
            wn = lerpf(1.0f, wn, k);
            wr = lerpf(1.0f, wr, k);
            bool inS = uvPrev.x > 0.0f && uvPrev.y > 0.0f && uvPrev.x < 1.0f && uvPrev.y < 1.0f;
            if (!inS) { wn = 1.0f; wr = 1.0f; }
            virtualHistoryNormalBasedConfidence = fminf(virtualHistoryNormalBasedConfidence, wn);
            virtualHistoryRoughnessBasedConfidence = fminf(virtualHistoryRoughnessBasedConfidence, wr);
        }

        const float virtualHistoryConfidenceForSmbRelaxation = virtualHistoryNormalBasedConfidence * virtualHistoryRoughnessBasedConfidence;
        const float virtualHistoryConfidence = virtualHistoryConfidenceForSmbRelaxation * virtualHistoryParallaxBasedConfidence;
        virtualHistoryAmount *= virtualHistoryRoughnessBasedConfidence;

        // surface-motion history
        const CatRomSetup smbSetup = SetupCatRom(smbSamplePos, c.gResourceSizeInvPrev, smbOcclusionWeights, smbAllowCatRom);
        f4 smbSpecHistory = ResolveCatRom4(smbSetup, a.histSpec);
        const float smbSpecFastHistory = ResolveBilinearCustom1(smbSetup, a.histSpecFast, smbOcclusionWeights);

        const float smcModified = SpecMagicCurve(roughnessModified); // used twice below
        float surfaceHistoryConfidence;
        {
            float ang = atanf(smbParallaxInPixelsMax * pixelSize / lengthX);
            float nonLinearAccumSpeed = 1.0f / (1.0f + smbSpecAccumSpeed);
            float h = lerpf(smbSpecHistory.w, spec.w, nonLinearAccumSpeed) * hitDistNormalization;
            float tana0 = LobeTanHalfAngle(roughnessModified, kLobeVolume);
            tana0 *= lerpf(NoV, 1.0f, roughnessModified);
            tana0 *= nonLinearAccumSpeed;
            tana0 /= saturate(h / frustumSize) + kEps;
            float a0 = fmaxf(atanf(tana0), kNormalEncodingError);
            float f = LinearStep(a0, 0.0f, ang);
            surfaceHistoryConfidence = (f * f) * (f * f); // Pow01(f, 4): f is already saturated
        }

        f2 maxResponsiveFrameNum;
        {
            float responsiveFactor = SmoothStep01((roughness + kEps) / (c.gResponsiveAccumulationRoughnessThreshold + kEps));
            float smc = smcModified;
            float fx = dot(N, normalize(smbNavg)), fy = dot(N, vmbN);
            float e = lerpf(32.0f, 1.0f, smc) * (1.0f - responsiveFactor), k = lerpf(smc, 1.0f, responsiveFactor);
            fx = k * Pow01(fx, e); // not the fast exp2(e log2 x): fx and fy are nearly equal and the ORDER of the two results selects a branch below
            fy = k * Pow01(fy, e);
            maxResponsiveFrameNum = mk2(fmaxf(c.gMaxAccumulatedFrameNum * fx, c.gHistoryFixFrameNum), fmaxf(c.gMaxAccumulatedFrameNum * fy, c.gHistoryFixFrameNum));
        }

        float smbMaxFrameNum = fminf(c.gMaxAccumulatedFrameNum * surfaceHistoryConfidence, maxResponsiveFrameNum.x);
        float smbBoostedMaxFrameNum = fmaxf(smbMaxFrameNum, c.gHistoryFixFrameNum * (1.0f - virtualHistoryConfidenceForSmbRelaxation));
        float smbSpecAccumSpeedBoosted = fminf(smbSpecAccumSpeed, smbBoostedMaxFrameNum);
        float vmbMaxFrameNum = fminf(c.gMaxAccumulatedFrameNum * virtualHistoryConfidence, maxResponsiveFrameNum.y);
        smbSpecAccumSpeed = fminf(smbSpecAccumSpeed, smbMaxFrameNum);
        vmbSpecAccumSpeed = fminf(vmbSpecAccumSpeed, vmbMaxFrameNum);

        float magic = vmbSpecAccumSpeed > smbSpecAccumSpeed ? 8.0f : 0.5f;
        virtualHistoryAmount *= 1.0f + (vmbSpecAccumSpeed - smbSpecAccumSpeed) / (magic * fmaxf(vmbSpecAccumSpeed, smbSpecAccumSpeed) + 1.0f);
        virtualHistoryAmount = saturate(virtualHistoryAmount);

        // virtual-motion history
        const f2 vmbSamplePos = mk2(saturate(vmbPixelUv.x) * c.gRectSizePrev[0], saturate(vmbPixelUv.y) * c.gRectSizePrev[1]);
        const CatRomSetup vmbSetup = SetupCatRom(vmbSamplePos, c.gResourceSizeInvPrev, vmbOcclusionWeights, vmbAllowCatRom);
        f4 vmbSpecHistory = ResolveCatRom4(vmbSetup, a.histSpec);
        const float vmbSpecFastHistory = ResolveBilinearCustom1(vmbSetup, a.histSpecFast, vmbOcclusionWeights);

        smbSpecHistory = ClampNegativeToZero(smbSpecHistory);
        vmbSpecHistory = ClampNegativeToZero(vmbSpecHistory);

        float smbNl = 1.0f / (1.0f + smbSpecAccumSpeed), vmbNl = 1.0f / (1.0f + vmbSpecAccumSpeed);
        // checkerboarded input: a pixel whose value was resolved from its neighbours accumulates slower (:731-735)
        const bool specHasData = !GENERAL || c.gSpecCheckerboard == 2u || checkerboard == c.gSpecCheckerboard;
        if (!specHasData)
        {
            smbNl *= lerpf(1.0f - c.gCheckerboardResolveAccumSpeed, 1.0f, smbNl);
            vmbNl *= lerpf(1.0f - c.gCheckerboardResolveAccumSpeed, 1.0f, vmbNl);
        }
        const float minHitNl = 1.0f / (1.0f + 0.5f * smcModified * c.gMaxAccumulatedFrameNum);
        f4 smbSpec = lerp4(smbSpecHistory, spec, smbNl);
        smbSpec.w = lerpf(smbSpecHistory.w, spec.w, fmaxf(smbNl, minHitNl));
        f4 vmbSpec = lerp4(vmbSpecHistory, spec, vmbNl);
        vmbSpec.w = lerpf(vmbSpecHistory.w, spec.w, fmaxf(vmbNl, minHitNl));
        f4 specResult = lerp4(smbSpec, vmbSpec, virtualHistoryAmount);
        specAccumSpeed = lerpf(smbSpecAccumSpeedBoosted, vmbSpecAccumSpeed, virtualHistoryAmount);
        const f4 specHistory = lerp4(smbSpecHistory, vmbSpecHistory, virtualHistoryAmount);

        // firefly suppressor
        const float specMaxRelativeIntensity = c.gFireflySuppressorMinRelativeScale + 38.0f / (specAccumSpeed + 1.0f);
        float specAntifireflyFactor = specAccumSpeed * c.gMaxBlurRadius * 0.1f;
        specAntifireflyFactor /= 1.0f + specAntifireflyFactor;
        float specLumaClamped = fminf(specResult.x, specHistory.x * specMaxRelativeIntensity);
        specLumaClamped = lerpf(specResult.x, specLumaClamped, specAntifireflyFactor);
        specResult = ChangeLuma(specResult, specLumaClamped);
        StoreRGBA16F(a.outSpec, x, y, specResult);

        // fast history
        float smbFastNl = fmaxf(1.0f - surfaceHistoryConfidence, 1.0f / (1.0f + fminf(smbSpecAccumSpeed, c.gMaxFastAccumulatedFrameNum)));
        float vmbFastNl = fmaxf(1.0f - virtualHistoryConfidence, 1.0f / (1.0f + fminf(vmbSpecAccumSpeed, c.gMaxFastAccumulatedFrameNum)));
        if (!specHasData)
        {
            smbFastNl *= lerpf(1.0f - c.gCheckerboardResolveAccumSpeed, 1.0f, smbFastNl);
            vmbFastNl *= lerpf(1.0f - c.gCheckerboardResolveAccumSpeed, 1.0f, vmbFastNl);
        }
        float smbSpecFast = lerpf(smbSpecFastHistory, spec.x, smbFastNl), vmbSpecFast = lerpf(vmbSpecFastHistory, spec.x, vmbFastNl);
        float specFastResult = lerpf(smbSpecFast, vmbSpecFast, virtualHistoryAmount);
        float specFastClamped = fminf(specFastResult, specHistory.x * specMaxRelativeIntensity * 4.0f);
        specFastResult = lerpf(specFastResult, specFastClamped, specAntifireflyFactor);
        StoreR16F(a.outSpecFast, x, y, specFastResult);
    }

    // Data2 is R32_UINT when there is a specular signal, R8_UINT (only the 4 surface-motion bits are non-zero) otherwise
    if (SPEC) StoreU32(a.outData2, x, y, PackData2(fbits, curvature, virtualHistoryAmount));
    else StoreU8(a.outData2, x, y, min(PackData2(fbits, curvature, virtualHistoryAmount), 255u));

    if (DIFF)
    {
        float diffHistoryConfidence = smbFootprintQuality;
        if (hasConfidence) diffHistoryConfidence *= LoadR8Unorm(Near(a.diffConfidence), x, y);
        diffAccumSpeed *= lerpf(diffHistoryConfidence, 1.0f, 1.0f / (1.0f + diffAccumSpeed));
        diffAccumSpeed = fminf(diffAccumSpeed, c.gMaxAccumulatedFrameNum);
        const f4 diff = LoadRGBA16F(Near(a.inDiff), x, y);

        const CatRomSetup smbSetup = SetupCatRom(smbSamplePos, c.gResourceSizeInvPrev, smbOcclusionWeights, smbAllowCatRom);
        f4 smbDiffHistory = ClampNegativeToZero(ResolveCatRom4(smbSetup, a.histDiff));
        const float smbDiffFastHistory = ResolveBilinearCustom1(smbSetup, a.histDiffFast, smbOcclusionWeights);

        float nl = 1.0f / (1.0f + diffAccumSpeed);
        const bool diffHasData = !GENERAL || c.gDiffCheckerboard == 2u || checkerboard == c.gDiffCheckerboard;
        if (!diffHasData) nl *= lerpf(1.0f - c.gCheckerboardResolveAccumSpeed, 1.0f, nl);
        const float minHitNl = 1.0f / (1.0f + 0.5f * __ldg(&a.lut[1023]).x * c.gMaxAccumulatedFrameNum); // SpecMagicCurve(1)
        f4 diffResult = lerp4(smbDiffHistory, diff, nl);
        diffResult.w = lerpf(smbDiffHistory.w, diff.w, fmaxf(nl, minHitNl));

        const float diffMaxRelativeIntensity = c.gFireflySuppressorMinRelativeScale + 38.0f / (diffAccumSpeed + 1.0f);
        float diffAntifireflyFactor = diffAccumSpeed * c.gMaxBlurRadius * 0.1f;
        diffAntifireflyFactor /= 1.0f + diffAntifireflyFactor;
        float diffLumaClamped = fminf(diffResult.x, smbDiffHistory.x * diffMaxRelativeIntensity);
        diffLumaClamped = lerpf(diffResult.x, diffLumaClamped, diffAntifireflyFactor);
        diffResult = ChangeLuma(diffResult, diffLumaClamped);
        StoreRGBA16F(a.outDiff, x, y, diffResult);

        float fastNl = 1.0f / (1.0f + fminf(diffAccumSpeed, c.gMaxFastAccumulatedFrameNum));
        if (!diffHasData) fastNl *= lerpf(1.0f - c.gCheckerboardResolveAccumSpeed, 1.0f, fastNl);
        float diffFastResult = lerpf(smbDiffFastHistory, diff.x, fastNl);
        float diffFastClamped = fminf(diffFastResult, smbDiffHistory.x * diffMaxRelativeIntensity * 4.0f);
        diffFastResult = lerpf(diffFastResult, diffFastClamped, diffAntifireflyFactor);
        StoreR16F(a.outDiffFast, x, y, diffFastResult);
    }
    else
        diffAccumSpeed = 0.0f;

    // PackData1
    if (DIFF && SPEC) StoreRG8Unorm(a.outData1, x, y, mk2(__fdiv_rn(diffAccumSpeed, kMaxAccum), __fdiv_rn(specAccumSpeed, kMaxAccum)));
    else StoreR8Unorm(a.outData1, x, y, __fdiv_rn(DIFF ? diffAccumSpeed : specAccumSpeed, kMaxAccum));
}

// =============================================================================================
// History fix
// =============================================================================================
struct HfArgs
{
    ReblurConstants c;
    Surf tiles, nr, data1, z, inDiff, inSpec, inDiffFast, inSpecFast, outDiff, outSpec, outDiffFast, outSpecFast;
    Surf guide;
    const float4* lut;
    int rowBegin, rowEnd;
    int useTma; // the fast-history window is staged by TMA (else by clamped loads)
    int perf;   // REBLUR_PERFORMANCE_MODE (REBLUR_HistoryFix.hlsli:88-90, :139-141; anti-firefly radius 3)
};

template <bool BOTH> __device__ __forceinline__ f2 LoadFrames(const Surf& s, int x, int y)
{
    if (BOTH)
    {
        f2 d = LoadRG8Unorm(s, x, y);
        return mk2(d.x * kMaxAccum, d.y * kMaxAccum);
    }
    float d = LoadR8Unorm(s, x, y) * kMaxAccum;
    return mk2(d, d);
}

// fast-history tile of the CTA: 32 x 8 texels + 2 of halo.  A TMA box must START on a 16-byte boundary of the row (8 texels of
// R16F; a start at tile - 2 faults with "illegal instruction", tools/tma_probe.cu) and hold whole 16-byte units: the box begins
// kHfPad = 8 texels left of the tile and is 48 texels wide, the kernel reads its columns 6..41.
constexpr int kHfBorder = 2, kHfPad = 8, kHfBoxW = 32 + 2 * kHfPad, kHfBoxH = 8 + 2 * kHfBorder;

// ---- sparse reconstruction of young history (REBLUR_HistoryFix.hlsli:63-167 / :268-371) -------------------------------------------
// Only pixels whose history is younger than gHistoryFixFrameNum frames run the 20-tap reconstruction: in steady state that is ~6 % of
// the specular and ~1 % of the diffuse pixels (disocclusions), but they are spread over ~20 % of the warps -- evaluated per pixel,
// every such warp walks the 20 taps with one or two live lanes.  The CTA therefore collects its (pixel, signal) items in shared
// memory and spreads item x tap tasks over all 256 threads; the pixel that owns an item then sums its 20 taps in the reference's tap
// order, so the result does not depend on which thread evaluated a tap.  CTAs with more than kHfMaxItems items (the first frames,
// where every pixel is young and no lane idles) keep the per-pixel loop.
struct HfItem
{
    int x, y, stridei, isSpec, perf;
    float stride, u, v;                  // pixelUv
    float Nvx, Nvy, Nvz, geoA, geoB;     // plane-distance weight
    float Nx, Ny, Nz, material;          // material = max(materialID, minMaterial)
    float minMaterial, normalParam, rrpx, rrpy, roughness;
    float hitDistScale, hitDist, hpx, hpy, frustumSize;
};
struct HfTap
{
    float w;
    unsigned lo, hi; // the tap's RGBA16F texel as loaded (12-byte records in shared memory)
};
constexpr int kHfTaps = 20, kHfMaxItems = 64;
// taps (i, j), j-major, centre and the four corners skipped: the reference's loop order
__constant__ signed char kHfTapI[kHfTaps] = {-1, 0, 1, -2, -1, 0, 1, 2, -2, -1, 1, 2, -2, -1, 0, 1, 2, -1, 0, 1};
__constant__ signed char kHfTapJ[kHfTaps] = {-2, -2, -2, -1, -1, -1, -1, -1, 0, 0, 0, 0, 1, 1, 1, 1, 1, 2, 2, 2};

// stride of the reconstruction of one signal; 0 = history old enough, nothing to do
template <bool IS_SPEC> __device__ __forceinline__ float HfStride(const ReblurConstants& c, float strideBase, float fn, float smc)
{
    float stride = strideBase * (fn < c.gHistoryFixFrameNum ? 1.0f : 0.0f);
    if (IS_SPEC) stride *= lerpf(0.5f, 1.0f, smc);
    return floorf(stride);
}

template <bool IS_SPEC>
__device__ __forceinline__ HfItem HfMakeItem(const HfArgs& a, int x, int y, float stride, float sigW, float viewZ, const Guide& g0, f3 Nv, f3 Xv, f2 pixelUv, float frustumSize, float fn)
{
    const ReblurConstants& c = a.c;
    HfItem it;
    it.x = x;
    it.y = y;
    it.stridei = (int)(stride + 0.5f);
    it.isSpec = IS_SPEC ? 1 : 0;
    it.perf = a.perf;
    it.stride = stride;
    it.u = pixelUv.x;
    it.v = pixelUv.y;
    const float nl = 1.0f / (1.0f + fn);
    const float roughness = g0.roughness, smc = g0.smc;
    it.minMaterial = IS_SPEC ? c.gSpecMinMaterial : c.gDiffMinMaterial;
    it.normalParam = NormalWeightParam(nl, c.gLobeAngleFraction, IS_SPEC ? roughness : 1.0f);
    it.geoA = 1.0f / (c.gPlaneDistSensitivity * frustumSize);
    it.geoB = -dot(Nv, Xv) * it.geoA;
    it.Nvx = Nv.x; it.Nvy = Nv.y; it.Nvz = Nv.z;
    it.Nx = g0.N.x; it.Ny = g0.N.y; it.Nz = g0.N.z;
    it.material = fmaxf(g0.materialID, it.minMaterial);
    const f2 rrp = RelaxedRoughnessWeightParams(roughness * roughness, sqrtf(c.gRoughnessFraction));
    it.rrpx = rrp.x; it.rrpy = rrp.y;
    it.roughness = roughness;
    it.hitDistScale = (c.gHitDistParams[0] + viewZ * c.gHitDistParams[1]) * (IS_SPEC ? g0.hitK : __ldg(&a.lut[1023]).y);
    it.hitDist = sigW * it.hitDistScale;
    const float hitDistFactor = saturate(it.hitDist / frustumSize);
    const f2 hp = HitDistanceWeightParams(hitDistFactor, nl, IS_SPEC ? smc : __ldg(&a.lut[1023]).x);
    it.hpx = hp.x; it.hpy = hp.y;
    it.frustumSize = frustumSize;
    return it;
}

// one tap of one item: weight and texel (isSpec is a compile-time constant on the per-pixel path)
template <bool BOTH>
__device__ __forceinline__ HfTap HfEvalTap(const ReblurConstants& c, const HfItem& it, bool isSpec, int i, int j, const Surf& zS, const Surf& nrS, const Surf& guideS,
                                           const Surf& data1S, const Surf& sigS)
{
    const int maxX = c.gRectSizeMinusOne[0], maxY = c.gRectSizeMinusOne[1];
    // uv for the in-screen test / view position is NOT clamped, the texel is
    const float u = __fadd_rn(it.u, __fmul_rn(__fmul_rn((float)i, it.stride), c.gRectSizeInv[0]));
    const float v = __fadd_rn(it.v, __fmul_rn(__fmul_rn((float)j, it.stride), c.gRectSizeInv[1]));
    const int px = clampi(it.x + i * it.stridei, 0, maxX), py = clampi(it.y + j * it.stridei, 0, maxY);
    const Guide gs = LoadGuide(guideS, nrS, px, py);
    const float zs = fabsf(LoadR32F(zS, px, py) * c.gViewZScale);
    const f3 Xvs = ReconstructViewPosition(mk2(u, v), c.gFrustum, zs, c.gOrthoMode);
    float w = (u > 0.0f && v > 0.0f && u < 1.0f && v < 1.0f) ? 1.0f : 0.0f;
    w *= NonExpWeight(it.Nvx * Xvs.x + it.Nvy * Xvs.y + it.Nvz * Xvs.z, it.geoA, it.geoB);
    w *= it.material == fmaxf(gs.materialID, it.minMaterial) ? 1.0f : 0.0f;
    w *= ExpWeight(AcosApprox(gs.N.x * it.Nx + gs.N.y * it.Ny + gs.N.z * it.Nz), it.normalParam, 0.0f);
    if (isSpec) w *= ExpWeight(gs.roughness * gs.roughness, it.rrpx, it.rrpy);
    if (!it.perf)
    {
        const f2 fr = LoadFrames<BOTH>(data1S, px, py);
        w *= 1.0f + (isSpec ? fr.y : fr.x);
    }
    HfTap t;
    t.lo = t.hi = 0u;
    if (w != 0.0f)
    {
        const uint2 sv = __ldg(TexelPtr<uint2>(sigS, px, py));
        t.lo = sv.x;
        t.hi = sv.y;
        const float hs = __half2float(__ushort_as_half((unsigned short)(sv.y >> 16))) * it.hitDistScale;
        w *= ExpWeight(saturate(hs / it.frustumSize), it.hpx, it.hpy);
        if (isSpec)
        {
            const float d = fabsf(it.hitDist - hs) / (fmaxf(it.hitDist, hs) + 0.001f);
            const float b = LinearStep(0.03f, 0.05f, it.roughness);
            w *= SmoothStep(0.2f + b, 0.05f + b, d);
        }
    }
    t.w = w;
    return t;
}
template <bool BOTH> __device__ __forceinline__ HfTap HfEvalTapAnywhere(const HfArgs& a, const HfItem& it, bool isSpec, int k)
{
    const int i = kHfTapI[k], j = kHfTapJ[k];
    const Surf& sig = isSpec ? a.inSpec : a.inDiff;
    // the 20 taps reach +-2 strides: one owner test for all of them
    if (FootprintLocal(a.z, it.y - 2 * it.stridei, it.y + 2 * it.stridei)) return HfEvalTap<BOTH>(a.c, it, isSpec, i, j, Near(a.z), Near(a.nr), Near(a.guide), Near(a.data1), Near(sig));
    return HfEvalTap<BOTH>(a.c, it, isSpec, i, j, a.z, a.nr, a.guide, a.data1, sig);
}

// the rest of the pass for one signal of one pixel: sum the taps (from shared memory, or evaluated here), fast-history clamp, stores
template <bool IS_SPEC, bool BOTH>
__device__ __forceinline__ void HistoryFixSignal(const HfArgs& a, int x, int y, const Surf& inSig, const Surf& inFast, const __half (*sFast)[kHfBoxW], const Surf& outSig,
                                                 const Surf& outFast, float viewZ, const Guide& g0, f3 Nv, f3 Xv, f2 pixelUv, float frustumSize, float fn, float stride,
                                                 const HfTap* taps)
{
    const ReblurConstants& c = a.c;
    const int maxX = c.gRectSizeMinusOne[0], maxY = c.gRectSizeMinusOne[1];
    f4 sig = LoadRGBA16F(Near(inSig), x, y);
    const float smc = g0.smc;

    if (stride != 0.0f)
    {
        float sum = 1.0f + fn;
        if (a.perf) sum = 1.0f + 1.0f / (1.0f + c.gMaxAccumulatedFrameNum) - 1.0f / (1.0f + fn);
        const float sigW = sig.w;
        sig = sig * sum;
        if (taps)
        {
#pragma unroll 4
            for (int k = 0; k < kHfTaps; k++)
            {
                const HfTap t = taps[k];
                if (t.w != 0.0f)
                {
                    sum += t.w;
                    sig = sig + UnpackHalf4(make_uint2(t.lo, t.hi)) * t.w;
                }
            }
        }
        else
        {
            const HfItem it = HfMakeItem<IS_SPEC>(a, x, y, stride, sigW, viewZ, g0, Nv, Xv, pixelUv, frustumSize, fn);
            for (int k = 0; k < kHfTaps; k++)
            {
                const HfTap t = HfEvalTapAnywhere<BOTH>(a, it, IS_SPEC, k);
                if (t.w != 0.0f)
                {
                    sum += t.w;
                    sig = sig + UnpackHalf4(make_uint2(t.lo, t.hi)) * t.w;
                }
            }
        }
        sig = sig * PositiveRcp(sum);
    }

    // 5x5 moments of the fast history from the staged tile (clamp-to-edge was patched into its halo): LDS with constant offsets
    const int cx = threadIdx.x + kHfPad, cy = threadIdx.y + kHfBorder;
    float center = __half2float(sFast[cy][cx]);
    float m1 = 0.0f, m2 = 0.0f;
#pragma unroll
    for (int j = -2; j <= 2; j++)
#pragma unroll
        for (int i = -2; i <= 2; i++)
        {
            float d = __half2float(sFast[cy + j][cx + i]);
            m1 += d;
            m2 += d * d;
        }
    float f = saturate(fn / (c.gHistoryFixFrameNum + kEps));
    if (IS_SPEC) f = lerpf(1.0f, f, smc);
    StoreR16F(outFast, x, y, lerpf(sig.x, center, f));

    float luma = sig.x;
    if (c.gAntiFirefly != 0.0f)
    {
        float am1 = 0.0f, am2 = 0.0f;
        const int R = a.perf ? 3 : 4; // REBLUR_ANTI_FIREFLY_FILTER_RADIUS
        for (int j = -R; j <= R; j++)
            for (int i = -R; i <= R; i++)
            {
                if (abs(i) <= 1 && abs(j) <= 1) continue;
                float d = LoadR16F(Near(inFast), clampi(x + i, 0, maxX), clampi(y + j, 0, maxY)); // +-4 rows
                am1 += d;
                am2 += d * d;
            }
        const float invNorm = a.perf ? 1.0f / 40.0f : 1.0f / 72.0f; // (2R + 1)^2 - 9 texels
        am1 *= invNorm;
        am2 *= invNorm;
        float sigma = GetStdDev(am1, am2) * 2.0f;
        luma = clampf(luma, am1 - sigma, am1 + sigma);
    }
    m1 *= 1.0f / 25.0f;
    m2 *= 1.0f / 25.0f;
    float sigma = GetStdDev(m1, m2) * 2.0f;
    float lumaClamped = clampf(luma, m1 - sigma, m1 + sigma);
    luma = lerpf(lumaClamped, luma, 1.0f / (1.0f + (c.gMaxFastAccumulatedFrameNum < c.gMaxAccumulatedFrameNum ? 1.0f : 0.0f) * fn * 2.0f));
    StoreRGBA16F(outSig, x, y, ChangeLuma(sig, luma));
}

template <bool DIFF, bool SPEC>
#ifndef NRD_B200_HF_MIN_BLOCKS
#define NRD_B200_HF_MIN_BLOCKS 4 // <= 64 registers
#endif
__global__ void __launch_bounds__(256, NRD_B200_HF_MIN_BLOCKS)
    ReblurHistoryFixKernel(const __grid_constant__ HfArgs a, const __grid_constant__ CUtensorMap diffFastMap, const __grid_constant__ CUtensorMap specFastMap)
{
    // The CTA stages the fast-history window of both signals (tile + 2 texels of halo) with TMA bulk tensor copies on one
    // mbarrier: the 5x5 moments of every pixel are then 25 shared-memory loads at constant offsets instead of 25 clamped global ones.
    __shared__ __align__(128) __half sFastDiff[DIFF ? kHfBoxH : 1][kHfBoxW];
    __shared__ __align__(128) __half sFastSpec[SPEC ? kHfBoxH : 1][kHfBoxW];
    __shared__ __align__(8) uint64_t bar;
    __shared__ HfItem sItems[kHfMaxItems];
    __shared__ HfTap sTaps[kHfMaxItems * kHfTaps];
    __shared__ int sCount;
    const ReblurConstants& c = a.c;
    const int tid = threadIdx.y * 32 + threadIdx.x;
    {
        const int boxX0 = blockIdx.x * 32 - kHfPad, boxY0 = a.rowBegin + blockIdx.y * 8 - kHfBorder;
        if (tid == 0) sCount = 0;
        if (a.useTma)
        {
            if (tid == 0) nrdb200_tma::BarrierInit(&bar);
            __syncthreads();
            if (tid == 0)
            {
                nrdb200_tma::BarrierExpect(&bar, (uint32_t)((DIFF ? sizeof(sFastDiff) : 0) + (SPEC ? sizeof(sFastSpec) : 0)));
                if (DIFF) nrdb200_tma::IssueTile2D(sFastDiff, &diffFastMap, boxX0, boxY0 - a.inDiffFast.ly0, &bar);
                if (SPEC) nrdb200_tma::IssueTile2D(sFastSpec, &specFastMap, boxX0, boxY0 - a.inSpecFast.ly0, &bar);
            }
        }
    }

    // per pixel: what the reconstruction needs, and whether it runs at all (while the tiles are in flight)
    const int x = blockIdx.x * 32 + threadIdx.x;
    const int y = a.rowBegin + blockIdx.y * 8 + threadIdx.y;
    bool active = x <= c.gRectSizeMinusOne[0] && y <= c.gRectSizeMinusOne[1] && y < a.rowEnd;
    if (active) active = LoadU8(Near(a.tiles), x >> 4, y >> 4) == 0;
    float viewZ = 0.0f;
    if (active)
    {
        viewZ = fabsf(LoadR32F(Near(a.z), x, y) * c.gViewZScale);
        active = viewZ <= c.gDenoisingRange;
    }
    Guide g0 = {};
    float frustumSize = 0.0f;
    f2 pixelUv = mk2(0.0f, 0.0f), frameNum = mk2(0.0f, 0.0f), stride = mk2(0.0f, 0.0f);
    f3 Xv = mk3(0.0f), Nv = mk3(0.0f);
    if (active)
    {
        g0 = LoadGuideLut(Near(a.guide), Near(a.nr), a.lut, x, y);
        frustumSize = c.gMinRectDimMulUnproject * lerpf(viewZ, 1.0f, fabsf(c.gOrthoMode));
        pixelUv = PixelUv(x, y, c.gRectSizeInv);
        Xv = ReconstructViewPosition(pixelUv, c.gFrustum, viewZ, c.gOrthoMode);
        Nv = RotateInverse(c.gViewToWorld, g0.N);
        frameNum = LoadFrames<DIFF && SPEC>(Near(a.data1), x, y);
        if (DIFF) stride.x = HfStride<false>(c, __fdiv_rn(c.gHistoryFixBasePixelStride, __fadd_rn(2.0f, frameNum.x)), frameNum.x, g0.smc);
        if (SPEC) stride.y = HfStride<true>(c, __fdiv_rn(c.gHistoryFixBasePixelStride, __fadd_rn(2.0f, frameNum.y)), frameNum.y, g0.smc);
    }
    __syncthreads(); // sCount = 0 is visible
    int slotD = -1, slotS = -1;
    if (DIFF && stride.x != 0.0f) slotD = atomicAdd(&sCount, 1);
    if (SPEC && stride.y != 0.0f) slotS = atomicAdd(&sCount, 1);
    __syncthreads();
    const int items = sCount;
    const bool compact = items > 0 && items <= kHfMaxItems; // the same decision in every thread of the CTA
    if (compact)
    {
        if (slotD >= 0) sItems[slotD] = HfMakeItem<false>(a, x, y, stride.x, LoadRGBA16F(Near(a.inDiff), x, y).w, viewZ, g0, Nv, Xv, pixelUv, frustumSize, frameNum.x);
        if (slotS >= 0) sItems[slotS] = HfMakeItem<true>(a, x, y, stride.y, LoadRGBA16F(Near(a.inSpec), x, y).w, viewZ, g0, Nv, Xv, pixelUv, frustumSize, frameNum.y);
        __syncthreads();
        for (int t = tid; t < items * kHfTaps; t += 256)
        {
            const int item = t / kHfTaps, k = t - item * kHfTaps;
            const HfItem it = sItems[item];
            sTaps[t] = HfEvalTapAnywhere<DIFF && SPEC>(a, it, it.isSpec != 0, k);
        }
    }

    // fast-history tiles
    {
        const int boxX0 = blockIdx.x * 32 - kHfPad, boxY0 = a.rowBegin + blockIdx.y * 8 - kHfBorder;
        if (a.useTma)
        {
            nrdb200_tma::BarrierWait(&bar, 0);
            if (DIFF) nrdb200_tma::PatchClampToEdge<__half, kHfBoxW, kHfBoxH>(sFastDiff, boxX0, boxY0, c.gRectSizeMinusOne[0], c.gRectSizeMinusOne[1], tid, 256);
            if (SPEC) nrdb200_tma::PatchClampToEdge<__half, kHfBoxW, kHfBoxH>(sFastSpec, boxX0, boxY0, c.gRectSizeMinusOne[0], c.gRectSizeMinusOne[1], tid, 256);
        }
        else
        {
            // same window staged with clamped loads (a surface TMA cannot address: base or pitch not 16-byte aligned; NRD_B200_NO_TMA=1)
            for (int i = tid; i < kHfBoxW * kHfBoxH; i += 256)
            {
                const int lx = i % kHfBoxW, ly = i / kHfBoxW;
                const int gx = clampi(boxX0 + lx, 0, c.gRectSizeMinusOne[0]), gy = clampi(boxY0 + ly, 0, c.gRectSizeMinusOne[1]);
                if (DIFF) sFastDiff[ly][lx] = __ushort_as_half((unsigned short)LoadU16(Near(a.inDiffFast), gx, gy));
                if (SPEC) sFastSpec[ly][lx] = __ushort_as_half((unsigned short)LoadU16(Near(a.inSpecFast), gx, gy));
            }
        }
        __syncthreads(); // tiles patched, taps of the compact path written
    }
    if (!active) return;

    if (DIFF)
        HistoryFixSignal<false, DIFF && SPEC>(a, x, y, a.inDiff, a.inDiffFast, sFastDiff, a.outDiff, a.outDiffFast, viewZ, g0, Nv, Xv, pixelUv, frustumSize, frameNum.x, stride.x,
                                              compact && slotD >= 0 ? &sTaps[slotD * kHfTaps] : nullptr);
    if (SPEC)
        HistoryFixSignal<true, DIFF && SPEC>(a, x, y, a.inSpec, a.inSpecFast, sFastSpec, a.outSpec, a.outSpecFast, viewZ, g0, Nv, Xv, pixelUv, frustumSize, frameNum.y, stride.y,
                                             compact && slotS >= 0 ? &sTaps[slotS * kHfTaps] : nullptr);
}

// =============================================================================================
// Temporal stabilization
// =============================================================================================
struct TsArgs
{
    ReblurConstants c;
    Surf tiles, nr, z, data1, data2, inDiff, inSpec, histDiffStab, histSpecStab, hitDist, mv;
    Surf baseColorMetalness; // IN_BASECOLOR_METALNESS (RGBA8), read only when the motion-vector patch is on (gSpecProbabilityThresholdsForMvModification.x < 1)
    Surf outInternal, outDiff, outSpec, outDiffStab, outSpecStab;
    Surf guide;
    const float4* lut;
    int rowBegin, rowEnd;
    int useTma; // the signal tiles are staged by TMA (else by clamped loads)
    int perf;   // REBLUR_PERFORMANCE_MODE: no CatRom, no rank clamp of the centre luma (REBLUR_TemporalStabilization.hlsli:118, :131-135)
};

__device__ __forceinline__ float Antilag(const ReblurConstants& c, float history, float avg, float sigma, float accumSpeed) // REBLUR_Common.hlsli:244-274, mode 2
{
    float s = sigma * c.gAntilagParams[0];
    float magic = c.gAntilagParams[1] * c.gFramerateScale * c.gFramerateScale;
    float hc = clampf(history, avg - s, avg + s);
    float d = fabsf(history - hc) / (fmaxf(history, hc) + kEps);
    return 1.0f / (1.0f + d * accumSpeed / magic);
}

// signal tile of the CTA: 32 x 8 texels of RGBA16F + 1 of halo.  The TMA box starts 2 texels (16 bytes) left of the tile (tma.cuh:
// the first byte of a box row must be 16-byte aligned) and is 36 texels wide; the kernel reads its columns 1..34.
constexpr int kTsPad = 2, kTsBoxW = 32 + 2 * kTsPad, kTsBoxH = 8 + 2;
__device__ __forceinline__ float TileLuma(uint2 t) { return __half2float(__ushort_as_half((unsigned short)(t.x & 0xFFFFu))); }

// 3x3 luma moments of a YCoCg signal from the staged tile (clamp-to-edge already in its halo).  sigma = sqrt(|m2 - m1^2|) cancels
// catastrophically on flat regions (the result is rounding noise of relative size ~3e-4 that then scales the clamping box), so the
// moments are accumulated in the oracle's order with individually rounded operations: centre first, then row-major, true division by 9.
__device__ __forceinline__ void LumaStats3x3(const uint2 (*tile)[kTsBoxW], float& luma, float& m1, float& m2, float& mn, float& mx)
{
    const int cx = threadIdx.x + kTsPad, cy = threadIdx.y + 1;
    luma = TileLuma(tile[cy][cx]);
    m1 = luma;
    m2 = __fmul_rn(luma, luma);
    mn = kInf;
    mx = -kInf;
#pragma unroll
    for (int j = -1; j <= 1; j++)
#pragma unroll
        for (int i = -1; i <= 1; i++)
        {
            if (i == 0 && j == 0) continue;
            float d = TileLuma(tile[cy + j][cx + i]);
            m1 = __fadd_rn(m1, d);
            m2 = __fadd_rn(m2, __fmul_rn(d, d));
            mn = fminf(mn, d);
            mx = fmaxf(mx, d);
        }
    m1 = __fdiv_rn(m1, 9.0f);
    m2 = __fdiv_rn(m2, 9.0f);
}
__device__ __forceinline__ float PinnedStdDev(float m1, float m2) { return __fsqrt_rn(fabsf(__fadd_rn(m2, -__fmul_rn(m1, m1)))); }

template <bool DIFF, bool SPEC>
__global__ void __launch_bounds__(256)
    ReblurTemporalStabilizationKernel(const __grid_constant__ TsArgs a, const __grid_constant__ CUtensorMap diffMap, const __grid_constant__ CUtensorMap specMap)
{
    // The CTA stages the signal window of both signals (tile + 1 texel of halo, whole RGBA16F texels) with TMA bulk tensor copies on
    // one mbarrier: the 3x3 luma moments and the centre texel of every pixel are shared-memory loads at constant offsets.
    __shared__ __align__(128) uint2 sDiff[DIFF ? kTsBoxH : 1][kTsBoxW];
    __shared__ __align__(128) uint2 sSpec[SPEC ? kTsBoxH : 1][kTsBoxW];
    __shared__ __align__(8) uint64_t bar;
    const ReblurConstants& c = a.c;
    const int x = blockIdx.x * 32 + threadIdx.x;
    const int y = a.rowBegin + blockIdx.y * 8 + threadIdx.y;
    const int maxX = c.gRectSizeMinusOne[0], maxY = c.gRectSizeMinusOne[1];
    {
        const int tid = threadIdx.y * 32 + threadIdx.x;
        const int boxX0 = blockIdx.x * 32 - kTsPad, boxY0 = a.rowBegin + blockIdx.y * 8 - 1;
        if (a.useTma)
        {
            if (tid == 0) nrdb200_tma::BarrierInit(&bar);
            __syncthreads();
            if (tid == 0)
            {
                // x of the copy in 32-bit words (2 per texel), y in rows held locally
                nrdb200_tma::BarrierExpect(&bar, (uint32_t)((DIFF ? sizeof(sDiff) : 0) + (SPEC ? sizeof(sSpec) : 0)));
                if (DIFF) nrdb200_tma::IssueTile2D(sDiff, &diffMap, boxX0 * 2, boxY0 - a.inDiff.ly0, &bar);
                if (SPEC) nrdb200_tma::IssueTile2D(sSpec, &specMap, boxX0 * 2, boxY0 - a.inSpec.ly0, &bar);
            }
            nrdb200_tma::BarrierWait(&bar, 0);
            if (DIFF) nrdb200_tma::PatchClampToEdge<uint2, kTsBoxW, kTsBoxH>(sDiff, boxX0, boxY0, maxX, maxY, tid, 256);
            if (SPEC) nrdb200_tma::PatchClampToEdge<uint2, kTsBoxW, kTsBoxH>(sSpec, boxX0, boxY0, maxX, maxY, tid, 256);
        }
        else
        {
            for (int i = tid; i < kTsBoxW * kTsBoxH; i += 256)
            {
                const int lx = i % kTsBoxW, ly = i / kTsBoxW;
                const int gx = clampi(boxX0 + lx, 0, maxX), gy = clampi(boxY0 + ly, 0, maxY);
                if (DIFF) sDiff[ly][lx] = __ldg(TexelPtr<uint2>(Near(a.inDiff), gx, gy));
                if (SPEC) sSpec[ly][lx] = __ldg(TexelPtr<uint2>(Near(a.inSpec), gx, gy));
            }
        }
        __syncthreads();
    }
    if (x > maxX || y > maxY || y >= a.rowEnd) return;
    if (LoadU8(Near(a.tiles), x >> 4, y >> 4) != 0) return;
    const float viewZ = fabsf(LoadR32F(Near(a.z), x, y) * c.gViewZScale);
    if (viewZ > c.gDenoisingRange) return;

    const f2 pixelUv = PixelUv(x, y, c.gRectSizeInv);
    const f3 Xv = ReconstructViewPosition(pixelUv, c.gFrustum, viewZ, c.gOrthoMode);
    const f3 X = PinnedRotate(c.gViewToWorld, Xv);

    const f4 mvRaw = LoadRGBA16F(Near(a.mv), x, y);
    f3 mv = mk3(__fmul_rn(mvRaw.x, c.gMvScale[0]), __fmul_rn(mvRaw.y, c.gMvScale[1]), __fmul_rn(mvRaw.z, c.gMvScale[2]));
    f3 Xprev = X;
    f2 smbPixelUv = mk2(__fadd_rn(pixelUv.x, mv.x), __fadd_rn(pixelUv.y, mv.y));
    if (c.gMvScale[3] == 0.0f)
    {
        if (c.gMvScale[2] == 0.0f) mv.z = __fadd_rn(PinnedRow(c.gWorldToViewPrev, 2, X.x, X.y, X.z), -viewZ);
        float viewZprev = __fadd_rn(viewZ, mv.z);
        f3 Xvprevlocal = ReconstructViewPosition(smbPixelUv, c.gFrustumPrev, viewZprev, c.gOrthoMode);
        f3 r = PinnedRotateInverse(c.gWorldToViewPrev, Xvprevlocal);
        Xprev = mk3(__fadd_rn(r.x, c.gCameraDelta[0]), __fadd_rn(r.y, c.gCameraDelta[1]), __fadd_rn(r.z, c.gCameraDelta[2]));
    }
    else
    {
        Xprev = mk3(__fadd_rn(X.x, mv.x), __fadd_rn(X.y, mv.y), __fadd_rn(X.z, mv.z));
        smbPixelUv = GetScreenUv(c.gWorldToClipPrev, Xprev);
    }

    const Guide g0 = LoadGuideLut(Near(a.guide), Near(a.nr), a.lut, x, y);
    f2 data1 = LoadFrames<DIFF && SPEC>(Near(a.data1), x, y);
    const unsigned d2 = SPEC ? LoadU32(Near(a.data2), x, y) : LoadU8(Near(a.data2), x, y);
    const unsigned bits = d2 & 0xFFu;
    const float virtualHistoryAmount = (float)((d2 >> 8) & 0xFFu) / 255.0f;
    const float curvature = __half2float(__ushort_as_half((unsigned short)(d2 >> 16)));

    const Bilinear smbF = GetBilinear(smbPixelUv, c.gRectSizePrev);
    const f4 smbOcclusion = mk4((bits & 1u) ? 1.0f : 0.0f, (bits & 2u) ? 1.0f : 0.0f, (bits & 4u) ? 1.0f : 0.0f, (bits & 8u) ? 1.0f : 0.0f);
    const f4 smbOcclusionWeights = CustomWeights(smbF, smbOcclusion);
    const bool smbAllowCatRom = (bits & 15u) == 15u && !a.perf;
    const float smbFootprintQuality = Sqrt01(ApplyBilinear(smbOcclusion.x, smbOcclusion.y, smbOcclusion.z, smbOcclusion.w, smbF));
    const f2 smbSamplePos = mk2(saturate(smbPixelUv.x) * c.gRectSizePrev[0], saturate(smbPixelUv.y) * c.gRectSizePrev[1]);
    const CatRomSetup smbSetup = SetupCatRom(smbSamplePos, c.gResourceSizeInvPrev, smbOcclusionWeights, smbAllowCatRom);

    if (DIFF)
    {
        float luma, m1, m2, mn, mx;
        LumaStats3x3(sDiff, luma, m1, m2, mn, mx);
        const float sigma = PinnedStdDev(m1, m2);
        if (c.gMaxBlurRadius != 0.0f && !a.perf) luma = clampf(luma, mn, mx);
        float history = fmaxf(ResolveCatRom1(smbSetup, a.histDiffStab), 0.0f);
        const float antilag = Antilag(c, history, m1, sigma, smbFootprintQuality * data1.x);
        const float tw = smbFootprintQuality * (data1.x / (1.0f + data1.x));
        float historyWeight = tw * antilag;
        historyWeight *= pixelUv.x >= c.gSplitScreen ? 1.0f : 0.0f;
        historyWeight *= smbPixelUv.x >= c.gSplitScreenPrev ? 1.0f : 0.0f;
        const float k = sigma * (1.0f + 3.0f * c.gFramerateScale * tw);
        history = clampf(history, m1 - k, m1 + k);
        const float stabilized = lerpf(luma, history, fminf(historyWeight, c.gStabilizationStrength));
        StoreRGBA16F(a.outDiff, x, y, ChangeLuma(UnpackHalf4(sDiff[threadIdx.y + 1][threadIdx.x + kTsPad]), stabilized));
        StoreR16F(a.outDiffStab, x, y, stabilized);
        data1.x += 1.0f;
        data1.x = lerpf(fminf(data1.x, c.gHistoryFixFrameNum), data1.x, antilag);
    }

    if (SPEC)
    {
        float luma, m1, m2, mn, mx;
        LumaStats3x3(sSpec, luma, m1, m2, mn, mx);
        const float sigma = PinnedStdDev(m1, m2);
        if (c.gMaxBlurRadius != 0.0f && !a.perf) luma = clampf(luma, mn, mx);

        f4 spec = UnpackHalf4(sSpec[threadIdx.y + 1][threadIdx.x + kTsPad]);
        float hitDistForTracking = spec.w * ((c.gHitDistParams[0] + viewZ * c.gHitDistParams[1]) * g0.hitK);
        if (c.gSpecPrepassBlurRadius != 0.0f) hitDistForTracking = fminf(hitDistForTracking, LoadR16F(Near(a.hitDist), x, y));

        const f3 V = c.gOrthoMode == 0.0f ? normalize(-X) : mk3(c.gViewVectorWorld[0], c.gViewVectorWorld[1], c.gViewVectorWorld[2]);
        const f3 Xvirtual = GetXvirtual(SetupXvirtual(curvature, length(X), g0.N, V, g0.aLog), hitDistForTracking, curvature, X, Xprev, g0.N, V);
        f2 vmbPixelUv = GetScreenUv(c.gWorldToClipPrev, Xvirtual);
        if (g0.materialID == c.gCameraAttachedReflectionMaterialID) vmbPixelUv = pixelUv;

        // modify MVs if requested (REBLUR_TemporalStabilization.hlsli:250-285): specular-dominant pixels get the motion of their reflection
        if (c.gSpecProbabilityThresholdsForMvModification[0] < 1.0f)
        {
            const float NoV = fabsf(dot(g0.N, V));
            const f4 bcm = UnpackRGBA8(LoadU32(Near(a.baseColorMetalness), x, y));
            // BRDF::ConvertBaseColorMetalnessToAlbedoRf0 / EnvironmentTerm_Rtg (MathLib, restated in oracle/mathlib.h)
            const float dielectric = saturate(1.0f - bcm.w);
            const f3 albedo = mk3(bcm.x * dielectric, bcm.y * dielectric, bcm.z * dielectric);
            const f3 Rf0 = lerp3(mk3(0.04f), xyz(bcm), bcm.w);
            const float m = g0.roughness * g0.roughness, m2r = m * m, m3r = m * m2r, n2 = NoV * NoV, n3 = NoV * n2;
            const float bias = ((0.99044f - 1.28514f * NoV) + (1.29678f - 0.755907f * NoV) * m) /
                               ((1.0f + 2.92338f * NoV + 59.4188f * n3) + (20.3225f - 27.0302f * NoV + 222.592f * n3) * m + (121.563f + 626.13f * NoV + 316.627f * n3) * m3r);
            const float scale = ((0.0365463f + 3.32707f * NoV) + (9.0632f - 9.04756f * NoV) * m) /
                                ((1.0f + 3.59685f * n2 - 1.36772f * n3) + (9.04401f - 16.3174f * n2 + 9.22949f * n3) * m + (5.56589f + 19.7886f * n2 - 20.2123f * n3) * m3r);
            (void)m2r;
            const f3 Fenv = mk3(saturate(Rf0.x * scale + bias), saturate(Rf0.y * scale + bias), saturate(Rf0.z * scale + bias));
            const float lumSpec = 0.2126f * Fenv.x + 0.7152f * Fenv.y + 0.0722f * Fenv.z;
            const float lumDiff = 0.2126f * albedo.x * (1.0f - Fenv.x) + 0.7152f * albedo.y * (1.0f - Fenv.y) + 0.0722f * albedo.z * (1.0f - Fenv.z);
            const float specProb = lumSpec / (lumDiff + lumSpec + kEps);
            float f = SmoothStep(c.gSpecProbabilityThresholdsForMvModification[0], c.gSpecProbabilityThresholdsForMvModification[1], specProb);
            f *= 1.0f - g0.smc;
            f *= 1.0f - Sqrt01(fabsf(curvature));
            if (f != 0.0f)
            {
                f3 specMv = Xvirtual - X;
                if (c.gMvScale[3] == 0.0f) specMv = mk3(vmbPixelUv.x - pixelUv.x, vmbPixelUv.y - pixelUv.y, PinnedRow(c.gWorldToViewPrev, 2, Xvirtual.x, Xvirtual.y, Xvirtual.z) - viewZ);
                const f3 newMv = mk3(specMv.x / c.gMvScale[0], specMv.y / c.gMvScale[1], c.gMvScale[2] == 0.0f ? mvRaw.z : specMv.z / c.gMvScale[2]);
                StoreRGBA16F(a.mv, x, y, mk4(lerp3(xyz(mvRaw), newMv, f), mvRaw.w));
            }
        }

        float smbHistory = ResolveCatRom1(smbSetup, a.histSpecStab);

        const Bilinear vmbF = GetBilinear(vmbPixelUv, c.gRectSizePrev);
        const f4 vmbOcclusion = mk4((bits & 16u) ? 1.0f : 0.0f, (bits & 32u) ? 1.0f : 0.0f, (bits & 64u) ? 1.0f : 0.0f, (bits & 128u) ? 1.0f : 0.0f);
        const f4 vmbOcclusionWeights = CustomWeights(vmbF, vmbOcclusion);
        const bool vmbAllowCatRom = (bits & 240u) == 240u && !a.perf;
        const float vmbFootprintQuality = Sqrt01(ApplyBilinear(vmbOcclusion.x, vmbOcclusion.y, vmbOcclusion.z, vmbOcclusion.w, vmbF));
        const f2 vmbSamplePos = mk2(saturate(vmbPixelUv.x) * c.gRectSizePrev[0], saturate(vmbPixelUv.y) * c.gRectSizePrev[1]);
        const CatRomSetup vmbSetup = SetupCatRom(vmbSamplePos, c.gResourceSizeInvPrev, vmbOcclusionWeights, vmbAllowCatRom);
        float vmbHistory = ResolveCatRom1(vmbSetup, a.histSpecStab);

        smbHistory = fmaxf(smbHistory, 0.0f);
        vmbHistory = fmaxf(vmbHistory, 0.0f);
        float history = lerpf(smbHistory, vmbHistory, virtualHistoryAmount);

        const float footprintQuality = lerpf(smbFootprintQuality, vmbFootprintQuality, virtualHistoryAmount);
        const float antilag = Antilag(c, history, m1, sigma, footprintQuality * data1.y);
        const float tw = footprintQuality * (data1.y / (1.0f + data1.y));
        float historyWeight = tw * antilag;
        historyWeight *= pixelUv.x >= c.gSplitScreen ? 1.0f : 0.0f;
        historyWeight *= virtualHistoryAmount != 1.0f ? (smbPixelUv.x >= c.gSplitScreenPrev ? 1.0f : 0.0f) : 1.0f;
        historyWeight *= virtualHistoryAmount != 0.0f ? (vmbPixelUv.x >= c.gSplitScreenPrev ? 1.0f : 0.0f) : 1.0f;

        const float responsiveFactor = SmoothStep01((g0.roughness + kEps) / (c.gResponsiveAccumulationRoughnessThreshold + kEps));
        const float smc = g0.smc;
        const float acceleration = lerpf(smc, 1.0f, 0.5f + responsiveFactor * 0.5f);
        historyWeight *= g0.materialID == c.gStrandMaterialID ? 0.5f : acceleration;

        const float k = sigma * (1.0f + 3.0f * c.gFramerateScale * tw);
        history = clampf(history, m1 - k, m1 + k);
        const float stabilized = lerpf(luma, history, fminf(historyWeight, c.gStabilizationStrength));
        StoreRGBA16F(a.outSpec, x, y, ChangeLuma(spec, stabilized));
        StoreR16F(a.outSpecStab, x, y, stabilized);
        data1.y += 1.0f;
        data1.y = lerpf(fminf(data1.y, c.gHistoryFixFrameNum), data1.y, antilag);
    }

    StoreU16(a.outInternal, x, y, PackInternalData(data1.x, data1.y, g0.materialID));
}

// =============================================================================================
// launchers
// =============================================================================================
template <bool DIFF, bool SPEC> static cudaError_t LaunchTa(const PassLaunch& p)
{
    TaArgs a;
    a.c = *(const ReblurConstants*)p.constants;
    a.guide = p.guide;
    a.lut = (const float4*)p.roughnessLut;
    Bindings b(p);
    a.tiles = b.Next(); a.nr = b.Next(); a.z = b.Next(); a.mv = b.Next();
    a.prevZ = b.Next(); a.prevNr = b.Next(); a.prevInternal = b.Next();
    a.mix = b.Next();                      // gIn_DisocclusionThresholdMix (bound to IN_VIEWZ when absent, never read then)
    a.diffConfidence = b.Next(DIFF);       // gIn_DiffConfidence
    a.specConfidence = b.Next(SPEC);       // gIn_SpecConfidence
    a.inDiff = b.Next(DIFF);
    a.inSpec = b.Next(SPEC);
    if (DIFF && SPEC) { a.histDiff = b.Next(); a.histSpec = b.Next(); a.histDiffFast = b.Next(); a.histSpecFast = b.Next(); }
    else { a.histDiff = b.Next(DIFF); a.histDiffFast = b.Next(DIFF); a.histSpec = b.Next(SPEC); a.histSpecFast = b.Next(SPEC); }
    a.prevHitDist = b.Next(SPEC); a.inHitDist = b.Next(SPEC);
    a.outDiff = b.Next(DIFF);
    a.outSpec = b.Next(SPEC);
    a.outDiffFast = b.Next(DIFF);
    a.outSpecFast = b.Next(SPEC); a.outHitDist = b.Next(SPEC);
    a.outData1 = b.Next();
    a.outData2 = b.Next();
    if (!b.Complete()) return cudaErrorInvalidValue;
    a.rowBegin = p.rowBegin;
    a.rowEnd = p.rowEnd;
    a.perf = p.kind.perf ? 1 : 0;
    const int W = (int)a.c.gRectSize[0];
    dim3 grid((W + 31) / 32, (p.rowEnd - p.rowBegin + 3) / 4), block(32, 4);
    // the switches ReblurTemporalAccumulationKernel<DIFF, SPEC> compiles as constants
    const ReblurConstants& c = a.c;
    const bool isDefault = !(DIFF && c.gDiffCheckerboard != 2u) && !(SPEC && c.gSpecCheckerboard != 2u) && c.gOrthoMode == 0.0f && c.gMvScale[3] == 0.0f &&
                           !c.gHasHistoryConfidence && !c.gHasDisocclusionThresholdMix && !(SPEC && c.gSpecPrepassBlurRadius == 0.0f) && !a.perf;
    if (!isDefault || p.preloadOnly) NRD_B200_LAUNCH(p, grid, block, a, ReblurTemporalAccumulationKernel<DIFF, SPEC, true>);
    if (isDefault || p.preloadOnly) NRD_B200_LAUNCH(p, grid, block, a, ReblurTemporalAccumulationKernel<DIFF, SPEC>);
    return cudaGetLastError();
}
cudaError_t LaunchReblurTemporalAccumulation(const PassLaunch& p)
{
    if (p.kind.signals == SIGNAL_DIFFUSE) return LaunchTa<true, false>(p);
    if (p.kind.signals == SIGNAL_SPECULAR) return LaunchTa<false, true>(p);
    return LaunchTa<true, true>(p);
}

template <bool DIFF, bool SPEC> static cudaError_t LaunchHf(const PassLaunch& p)
{
    HfArgs a;
    a.c = *(const ReblurConstants*)p.constants;
    a.guide = p.guide;
    a.lut = (const float4*)p.roughnessLut;
    Bindings b(p);
    a.tiles = b.Next(); a.nr = b.Next(); a.data1 = b.Next(); a.z = b.Next();
    a.inDiff = b.Next(DIFF);
    a.inSpec = b.Next(SPEC);
    a.inDiffFast = b.Next(DIFF);
    a.inSpecFast = b.Next(SPEC);
    a.outDiff = b.Next(DIFF);
    a.outSpec = b.Next(SPEC);
    a.outDiffFast = b.Next(DIFF);
    a.outSpecFast = b.Next(SPEC);
    if (!b.Complete()) return cudaErrorInvalidValue;
    a.rowBegin = p.rowBegin;
    a.rowEnd = p.rowEnd;
    a.perf = p.kind.perf ? 1 : 0;
    const int W = (int)a.c.gRectSize[0];
    dim3 grid((W + 31) / 32, (p.rowEnd - p.rowBegin + 7) / 8), block(32, 8);
    if (p.preloadOnly)
    {
        cudaFuncAttributes fa;
        return cudaFuncGetAttributes(&fa, ReblurHistoryFixKernel<DIFF, SPEC>);
    }
    // TMA descriptors of the two fast-history textures (pool textures: 256-byte aligned rows, device/tma.cuh)
    CUtensorMap diffMap, specMap;
    memset(&diffMap, 0, sizeof(diffMap));
    memset(&specMap, 0, sizeof(specMap));
    a.useTma = nrdb200_tma::Enabled() && (!DIFF || nrdb200_tma::MakeSurfaceMap16(a.inDiffFast, kHfBoxW, kHfBoxH, &diffMap)) &&
               (!SPEC || nrdb200_tma::MakeSurfaceMap16(a.inSpecFast, kHfBoxW, kHfBoxH, &specMap));
    ReblurHistoryFixKernel<DIFF, SPEC><<<grid, block, 0, p.stream>>>(a, diffMap, specMap);
    return cudaGetLastError();
}
cudaError_t LaunchReblurHistoryFix(const PassLaunch& p)
{
    if (p.kind.signals == SIGNAL_DIFFUSE) return LaunchHf<true, false>(p);
    if (p.kind.signals == SIGNAL_SPECULAR) return LaunchHf<false, true>(p);
    return LaunchHf<true, true>(p);
}

template <bool DIFF, bool SPEC> static cudaError_t LaunchTs(const PassLaunch& p)
{
    TsArgs a;
    a.c = *(const ReblurConstants*)p.constants;
    a.guide = p.guide;
    a.lut = (const float4*)p.roughnessLut;
    Bindings b(p);
    a.tiles = b.Next(); a.nr = b.Next();
    a.baseColorMetalness = b.Next(SPEC); // gIn_BaseColor_Metalness (bound to IN_VIEWZ when absent, never read then)
    a.z = b.Next(); a.data1 = b.Next(); a.data2 = b.Next();
    a.inDiff = b.Next(DIFF);
    a.inSpec = b.Next(SPEC);
    a.histDiffStab = b.Next(DIFF);
    a.histSpecStab = b.Next(SPEC); a.hitDist = b.Next(SPEC);
    a.mv = b.Next();
    a.outInternal = b.Next();
    a.outDiff = b.Next(DIFF);
    a.outSpec = b.Next(SPEC);
    a.outDiffStab = b.Next(DIFF);
    a.outSpecStab = b.Next(SPEC);
    if (!b.Complete()) return cudaErrorInvalidValue;
    a.rowBegin = p.rowBegin;
    a.rowEnd = p.rowEnd;
    a.perf = p.kind.perf ? 1 : 0;
    const int W = (int)a.c.gRectSize[0];
    dim3 grid((W + 31) / 32, (p.rowEnd - p.rowBegin + 7) / 8), block(32, 8);
    if (p.preloadOnly)
    {
        cudaFuncAttributes fa;
        return cudaFuncGetAttributes(&fa, ReblurTemporalStabilizationKernel<DIFF, SPEC>);
    }
    // TMA descriptors of the two signals (RGBA16F = 2 words per texel); user textures whose base or pitch is not 16-byte aligned
    // are staged with clamped loads instead
    CUtensorMap diffMap, specMap;
    memset(&diffMap, 0, sizeof(diffMap));
    memset(&specMap, 0, sizeof(specMap));
    a.useTma = nrdb200_tma::Enabled() && (!DIFF || nrdb200_tma::MakeSurfaceMap(a.inDiff, 2, kTsBoxW, kTsBoxH, &diffMap)) &&
               (!SPEC || nrdb200_tma::MakeSurfaceMap(a.inSpec, 2, kTsBoxW, kTsBoxH, &specMap));
    ReblurTemporalStabilizationKernel<DIFF, SPEC><<<grid, block, 0, p.stream>>>(a, diffMap, specMap);
    return cudaGetLastError();
}
cudaError_t LaunchReblurTemporalStabilization(const PassLaunch& p)
{
    if (p.kind.signals == SIGNAL_DIFFUSE) return LaunchTs<true, false>(p);
    if (p.kind.signals == SIGNAL_SPECULAR) return LaunchTs<false, true>(p);
    return LaunchTs<true, true>(p);
}

#if !defined(NRD_B200_NO_STRIPS)
cudaError_t SetPeerTableReblurTemporal(int slot, const PeerTable* table, const cudaStream_t* stream) { return SetPeerTableThisTU(slot, table, stream); }
#endif
} // namespace nrdb200
