// SIGMA_SHADOW / SIGMA_SHADOW_TRANSLUCENCY passes on sm_90a: ClassifyTiles, SmoothTiles, Copy, Blur / PostBlur, TemporalStabilization.
// The shadow signal is SIGMA_TYPE (SIGMA_Config.hlsli:38-43): a float in R8 textures, or -- translucent variant, template flag TR --
// a float4 {shadow, translucency.rgb} in RGBA8 textures fed by IN_TRANSLUCENCY.  The kernels are written once over sgt:: overloads.
// Semantics: reference Shaders/Include/SIGMA_ClassifyTiles.hlsli:10-81, SIGMA_SmoothTiles.hlsli:10-48, SIGMA_Copy.hlsli:10-24,
// SIGMA_Blur.hlsli:11-268, SIGMA_TemporalStabilization.hlsli:10-226, SIGMA_Common.hlsli:13-130 (default switches:
// 5x5 dense estimate, sparse 8-tap blur in screen space, NRD_FRAME rotators, CatRom history).
#include "reblur_math.cuh"
#include "launch.h"

#include <cstring>

namespace nrdb200
{
using namespace rb;

namespace sg
{
constexpr float kFp16Max = 65504.0f;
constexpr float kMaxPixelRadius = 32.0f;

__device__ __forceinline__ float KernelRadiusInPixels(float hitDist, float unprojectZ, float scale)
{
    float r = hitDist / unprojectZ * scale;
    return clampf(r, fminf(r, 2.0f), kMaxPixelRadius);
}
__device__ __forceinline__ bool IsLit(float p) { return p >= kFp16Max; }
__device__ __forceinline__ float BothLitOrUnlit(float a, float b) { return ((a == 0.0f) == (b == 0.0f)) ? 1.0f : 0.0f; }

// clamp-to-edge bilinear fetch of the RG8 smoothed-tiles texture
__device__ __forceinline__ f2 TilesTexel(const Surf& s, int x, int y) { return LoadRG8Unorm(s, clampi(x, 0, s.w - 1), clampi(y, 0, s.h - 1)); }
__device__ __forceinline__ f2 TilesLinear(const Surf& s, float u, float v)
{
    float px = u * (float)s.w - 0.5f, py = v * (float)s.h - 0.5f;
    float fx = floorf(px), fy = floorf(py), wx = px - fx, wy = py - fy;
    int x0 = (int)fx, y0 = (int)fy;
    f2 a = lerp2(TilesTexel(s, x0, y0), TilesTexel(s, x0 + 1, y0), wx);
    f2 b = lerp2(TilesTexel(s, x0, y0 + 1), TilesTexel(s, x0 + 1, y0 + 1), wx);
    return lerp2(a, b, wy);
}
// TextureCubic (SIGMA_Common.hlsli:46-95): B-spline bicubic through 4 bilinear taps
__device__ __forceinline__ void CubicAxis(float f, float& o0, float& o1, float& t)
{
    float f2 = f * f, f3 = f2 * f;
    const float k = 1.0f / 6.0f;
    float p0 = k * (-f3 + 3.0f * f2 - 3.0f * f + 1.0f), p1 = k * (3.0f * f3 - 6.0f * f2 + 4.0f);
    float p2 = k * (-3.0f * f3 + 3.0f * f2 + 3.0f * f + 1.0f), p3 = k * f3;
    o0 = 1.0f + f - p1 / (p0 + p1);
    o1 = 1.0f - f + p3 / (p2 + p3);
    t = p0 + p1;
}
__device__ __forceinline__ f2 TextureCubic(const Surf& s, float u, float v)
{
    float sx = (float)s.w, sy = (float)s.h;
    float fx = u * sx - 0.5f, fy = v * sy - 0.5f;
    fx -= floorf(fx);
    fy -= floorf(fy);
    float xo0, xo1, tx, yo0, yo1, ty;
    CubicAxis(fx, xo0, xo1, tx);
    CubicAxis(fy, yo0, yo1, ty);
    float u10 = u - xo0 / sx, u00 = u + xo1 / sx;   // uv_10_00.x / .z
    float vLo = v + yo1 / sy, vHi = v - yo0 / sy;   // uv_10_00.y (after -= yw.y * dxdy.w) / uv_11_01.y
    f2 c00 = TilesLinear(s, u00, vLo), c10 = TilesLinear(s, u10, vLo), c01 = TilesLinear(s, u00, vHi), c11 = TilesLinear(s, u10, vHi);
    c00 = lerp2(c00, c01, ty);
    c10 = lerp2(c10, c11, ty);
    return lerp2(c00, c10, tx);
}
} // namespace sg

// the shadow signal: float (opaque) or f4 (translucent); one set of overloads so that every kernel is written once
namespace sgt
{
template <bool TR> struct Sig { typedef float T; };
template <> struct Sig<true> { typedef f4 T; };
__device__ __forceinline__ float Splat(float v, float) { return v; }
__device__ __forceinline__ f4 Splat(float v, f4) { return mk4(v); }
__device__ __forceinline__ float X(float v) { return v; }
__device__ __forceinline__ float X(f4 v) { return v.x; }
__device__ __forceinline__ float Scale(float v, float w) { return v * w; }
__device__ __forceinline__ f4 Scale(f4 v, float w) { return v * w; }
__device__ __forceinline__ float Sq(float v) { return v * v; }
__device__ __forceinline__ f4 Sq(f4 v) { return v * v; }
__device__ __forceinline__ float Lerp(float a, float b, float t) { return lerpf(a, b, t); }
__device__ __forceinline__ f4 Lerp(f4 a, f4 b, float t) { return lerp4(a, b, t); }
__device__ __forceinline__ float Clamp(float v, float a, float b) { return clampf(v, a, b); }
__device__ __forceinline__ f4 Clamp(f4 v, f4 a, f4 b) { return mk4(clampf(v.x, a.x, b.x), clampf(v.y, a.y, b.y), clampf(v.z, a.z, b.z), clampf(v.w, a.w, b.w)); }
__device__ __forceinline__ float Sat(float v) { return saturate(v); }
__device__ __forceinline__ f4 Sat(f4 v) { return mk4(saturate(v.x), saturate(v.y), saturate(v.z), saturate(v.w)); }
__device__ __forceinline__ float Pack(float v) { return Sqrt01(v); } // PackShadow (SIGMA_Common.hlsli:13)
__device__ __forceinline__ f4 Pack(f4 v) { return mk4(Sqrt01(v.x), Sqrt01(v.y), Sqrt01(v.z), Sqrt01(v.w)); }
__device__ __forceinline__ float StdDev(float m1, float m2) { return GetStdDev(m1, m2); }
__device__ __forceinline__ f4 StdDev(f4 m1, f4 m2) { return mk4(GetStdDev(m1.x, m2.x), GetStdDev(m1.y, m2.y), GetStdDev(m1.z, m2.z), GetStdDev(m1.w, m2.w)); }
// texel access in the signal's storage format (R8_UNORM / RGBA8_UNORM)
__device__ __forceinline__ void Load(const Surf& s, int x, int y, float& v) { v = LoadR8Unorm(s, x, y); }
__device__ __forceinline__ void Load(const Surf& s, int x, int y, f4& v) { v = UnpackRGBA8(LoadU32(s, x, y)); }
__device__ __forceinline__ void Store(const Surf& s, int x, int y, float v) { StoreR8Unorm(s, x, y, v); }
__device__ __forceinline__ void Store(const Surf& s, int x, int y, f4 v) { StoreU32(s, x, y, PackRGBA8(v)); }
} // namespace sgt

// ---------------------------------------------------------------------------------------------
struct SigmaTilesArgs
{
    Surf z, penumbra, translucency, tiles;
    float viewZScale, denoisingRange, unproject, orthoMode;
    int tilesW, tilesH;
};

// one warp per 16x16 tile: 3 counters + max radius reduced with shuffles (no shared-memory atomics)
template <bool TR>
__global__ void __launch_bounds__(256) SigmaClassifyTilesKernel(const __grid_constant__ SigmaTilesArgs a)
{
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (warp >= a.tilesW * a.tilesH) return;
    const int tx = warp % a.tilesW, ty = warp / a.tilesW;
    if (ty < a.tiles.y0 || ty >= a.tiles.y1) return; // tile rows of another strip
    int nLit = 0, nUmbra = 0, nInf = 0;
    float maxRadius = 0.0f;
#pragma unroll
    for (int i = 0; i < 8; i++)
    {
        int idx = i * 32 + lane;
        int x = tx * 16 + (idx & 15), y = ty * 16 + (idx >> 4);
        // every texture reads 0 out of its own bounds: viewZ is read at rectOrigin + pixel (a view that ends earlier under dynamic
        // resolution), the penumbra and the translucency at the pixel itself
        const float h = Inside(a.penumbra, x, y) ? LoadR16F(a.penumbra, x, y) : 0.0f;
        const float z = Inside(a.z, x, y) ? LoadR32F(a.z, x, y) : 0.0f;
        bool isOpaque = true;
        if (TR) // SIGMA_ClassifyTiles.hlsli:45-48: luminance of the translucency colour (out-of-bounds loads read 0: opaque)
        {
            const f4 t = Inside(a.translucency, x, y) ? UnpackRGBA8(LoadU32(a.translucency, x, y)) : mk4(0.0f);
            isOpaque = (t.y * 0.2126f + t.z * 0.7152f + t.w * 0.0722f) < 0.003f;
        }
        float viewZ = fabsf(z * a.viewZScale);
        bool isInf = viewZ > a.denoisingRange, isShadow = h == 0.0f, isLit = sg::IsLit(h);
        nLit += (isLit || isInf || isShadow) ? 1 : 0;
        nUmbra += ((!isLit && isOpaque) || isInf || isShadow) ? 1 : 0;
        nInf += isInf ? 1 : 0;
        float hitDist = (isLit || isInf) ? 0.0f : h;
        float pixelSize = a.unproject * lerpf(viewZ, 1.0f, fabsf(a.orthoMode));
        maxRadius = fmaxf(maxRadius, sg::KernelRadiusInPixels(hitDist, pixelSize, 1.0f));
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1)
    {
        nLit += __shfl_xor_sync(0xffffffffu, nLit, o);
        nUmbra += __shfl_xor_sync(0xffffffffu, nUmbra, o);
        nInf += __shfl_xor_sync(0xffffffffu, nInf, o);
        maxRadius = fmaxf(maxRadius, __shfl_xor_sync(0xffffffffu, maxRadius, o));
    }
    if (lane == 0)
    {
        f4 r = mk4((nLit == 256 || nUmbra == 256) ? 0.0f : 1.0f, saturate(maxRadius / 16.0f), nInf == 256 ? 1.0f : 0.0f, 0.0f);
        StoreU32(a.tiles, tx, ty, PackRGBA8(r));
    }
}

struct SigmaSmoothArgs
{
    Surf tiles, smoothed;
    int tilesMaxX, tilesMaxY;
};

__global__ void __launch_bounds__(256) SigmaSmoothTilesKernel(const __grid_constant__ SigmaSmoothArgs a)
{
    const int x = blockIdx.x * 16 + threadIdx.x, y = blockIdx.y * 16 + threadIdx.y;
    if (!Inside(a.smoothed, x, y) || y < a.smoothed.y0 || y >= a.smoothed.y1) return;
    f4 center = UnpackRGBA8(LoadU32(a.tiles, x, y));
    float k = 1.01f / (center.y + 0.01f);
    float blurry = 0.0f, sum = 0.0f;
#pragma unroll
    for (int j = -1; j <= 1; j++)
#pragma unroll
        for (int i = -1; i <= 1; i++)
        {
            float d2 = (float)(i * i + j * j);
            float d = sqrtf(d2);
            float w = exp2f(-k * d * d);
            f4 t = UnpackRGBA8(LoadU32(a.tiles, clampi(x + i, 0, a.tilesMaxX), clampi(y + j, 0, a.tilesMaxY)));
            blurry += t.x * w;
            sum += w;
        }
    StoreRG8Unorm(a.smoothed, x, y, mk2(center.z, blurry / sum));
}

struct SigmaCopyArgs
{
    Surf tiles, inHistory, inLength, outHistory, outLength;
    int w, h, isRectChanged, rowBegin, rowEnd;
};

template <bool TR>
__global__ void __launch_bounds__(256) SigmaCopyKernel(const __grid_constant__ SigmaCopyArgs a)
{
    const int x = blockIdx.x * 32 + threadIdx.x, y = a.rowBegin + blockIdx.y * 8 + threadIdx.y;
    if (x >= a.w || y >= a.h || y >= a.rowEnd) return;
    if (LoadRG8Unorm(a.tiles, x >> 4, y >> 4).x != 0.0f && !a.isRectChanged) return;
    if (TR) StoreU32(a.outHistory, x, y, LoadU32(a.inHistory, x, y));
    else StoreU8(a.outHistory, x, y, LoadU8(a.inHistory, x, y));
    StoreU32(a.outLength, x, y, LoadU32(a.inLength, x, y));
}

// ---------------------------------------------------------------------------------------------
struct SigmaBlurArgs
{
    SigmaConstants c;
    Surf z, nr, penumbra, tiles, shadow, outPenumbra, outShadow;
    int rowBegin, rowEnd;
};

template <bool FIRST, bool TR>
__global__ void __launch_bounds__(256) SigmaBlurKernel(const __grid_constant__ SigmaBlurArgs a)
{
    typedef typename sgt::Sig<TR>::T S;
    const SigmaConstants& c = a.c;
    const int x = blockIdx.x * 32 + threadIdx.x, y = a.rowBegin + blockIdx.y * 8 + threadIdx.y;
    const int maxX = c.gRectSizeMinusOne[0], maxY = c.gRectSizeMinusOne[1];
    if (x > maxX || y > maxY || y >= a.rowEnd) return;
    if (LoadRG8Unorm(a.tiles, x >> 4, y >> 4).x != 0.0f) return;

    const float centerPenumbra = LoadR16F(a.penumbra, x, y);
    const float viewZ = fabsf(LoadR32F(a.z, x, y) * c.gViewZScale);
    if (viewZ > c.gDenoisingRange) return;

    // SIGMA_Blur.hlsli:24-34: the signal comes from a texture unless this is the first pass of the opaque variant; only the
    // second pass reads a packed (sqrt) value
    auto shadowAt = [&](int px, int py, float penum) -> S {
        if (FIRST && !TR) return sgt::Splat(sg::IsLit(penum) ? 1.0f : 0.0f, S());
        S s;
        sgt::Load(a.shadow, px, py, s);
        return FIRST ? s : sgt::Sq(s);
    };

    const f2 pixelUv = PixelUv(x, y, c.gRectSizeInv);
    const float tileValue = sg::TextureCubic(a.tiles, pixelUv.x * c.gResolutionScale[0], pixelUv.y * c.gResolutionScale[1]).y;
    if (tileValue == 0.0f || centerPenumbra == 0.0f)
    {
        StoreR16F(a.outPenumbra, x, y, centerPenumbra);
        sgt::Store(a.outShadow, x, y, sgt::Pack(shadowAt(x, y, centerPenumbra)));
        return;
    }

    const f3 Xv = ReconstructViewPosition(pixelUv, c.gFrustum, viewZ, c.gOrthoMode);
    const f3 N = DecodeGuide(LoadU32(a.nr, x, y)).N;
    const f3 Nv = Rotate(c.gWorldToView, N);
    const float pixelSize = c.gUnproject * lerpf(viewZ, 1.0f, fabsf(c.gOrthoMode));
    const float frustumSize = c.gMinRectDimMulUnproject * lerpf(viewZ, 1.0f, fabsf(c.gOrthoMode));
    const f3 Vv = c.gOrthoMode == 0.0f ? normalize(-Xv) : mk3(0.0f, 0.0f, -1.0f);
    const float NoV = fabsf(dot(Nv, Vv));
    const float geoA = 1.0f / (c.gPlaneDistSensitivity * frustumSize), geoB = -dot(Nv, Xv) * geoA;

    // dense 5x5: shadow filter + penumbra size estimate
    float sumX = 0.0f, sumY = 0.0f, penumbra = 0.0f;
    S result = sgt::Splat(0.0f, S()), centerTap = sgt::Splat(0.0f, S());
#pragma unroll
    for (int j = -2; j <= 2; j++)
#pragma unroll
        for (int i = -2; i <= 2; i++)
        {
            int px = clampi(x + i, 0, maxX), py = clampi(y + j, 0, maxY);
            float penum = LoadR16F(a.penumbra, px, py);
            S s = shadowAt(px, py, penum);
            float w = 1.0f;
            if (i == 0 && j == 0) centerTap = s;
            else
            {
                float zs = fabsf(LoadR32F(a.z, px, py) * c.gViewZScale);
                f2 uv = mk2(pixelUv.x + (float)i * c.gRectSizeInv[0], pixelUv.y + (float)j * c.gRectSizeInv[1]);
                f3 Xvs = ReconstructViewPosition(uv, c.gFrustum, zs, c.gOrthoMode);
                w = NonExpWeight(dot(Nv, Xvs), geoA, geoB);
                w *= sg::BothLitOrUnlit(centerPenumbra, penum);
                float r2 = (float)(i * i + j * j) * 0.25f; // (length(offset / BORDER))^2
                w *= __expf(-0.66f * r2);
            }
            if (w != 0.0f) result = result + sgt::Scale(s, w);
            sumX += w;
            w *= pixelSize / (pixelSize + penum);
            w *= sg::IsLit(penum) ? 0.0f : 1.0f;
            penumbra += w == 0.0f ? 0.0f : penum * w;
            sumY += w;
        }
    result = sgt::Scale(result, 1.0f / sumX);
    sumX = 1.0f;
    penumbra /= fmaxf(sumY, kEps);
    sumY = sumY != 0.0f ? 1.0f : 0.0f;

    float f = SmoothStep(0.0f, 2.0f, penumbra / pixelSize);
    result = sgt::Lerp(centerTap, result, f);
    f = lerpf(4.0f, 1.0f, f);
    result = sgt::Scale(result, f);
    penumbra *= f;
    sumX *= f;
    sumY *= f;

    // sparse 8-tap blur in screen space
    const float blurRadius = sg::KernelRadiusInPixels(penumbra, pixelSize, tileValue);
    const float* rot = FIRST ? c.gRotator : c.gRotatorPost;
    f2 skew = lerp2(mk2(1.0f - fabsf(Nv.x), 1.0f - fabsf(Nv.y)), mk2(1.0f, 1.0f), NoV);
    float m = fmaxf(skew.x, skew.y);
    skew = mk2(skew.x / m * (c.gRectSizeInv[0] * blurRadius), skew.y / m * (c.gRectSizeInv[1] * blurRadius));
    const f4 sr = mk4(rot[0] * skew.x, rot[1] * skew.x, rot[2] * skew.y, rot[3] * skew.y);
    const float invEstimatedPenumbra = 1.0f / fmaxf(penumbra, kEps);
    const float tapX[8] = {-1.0f, 0.0f, 1.0f, 0.0f, -0.35355339f, 0.35355339f, 0.35355339f, -0.35355339f};
    const float tapY[8] = {0.0f, 1.0f, 0.0f, -1.0f, 0.35355339f, 0.35355339f, -0.35355339f, -0.35355339f};
    const int W = (int)c.gRectSize[0], H = (int)c.gRectSize[1];
#pragma unroll
    for (int n = 0; n < 8; n++)
    {
        float u = __fadd_rn(pixelUv.x, __fadd_rn(__fmul_rn(tapX[n], sr.x), __fmul_rn(tapY[n], sr.y)));
        float v = __fadd_rn(pixelUv.y, __fadd_rn(__fmul_rn(tapX[n], sr.z), __fmul_rn(tapY[n], sr.w)));
        float fx = floorf(__fmul_rn(u, c.gRectSize[0])), fy = floorf(__fmul_rn(v, c.gRectSize[1]));
        int ix = (int)fx, iy = (int)fy;
        bool inScreen = (unsigned)ix < (unsigned)W && (unsigned)iy < (unsigned)H;
        int tx = clampi(ix, 0, W - 1), ty = clampi(iy, 0, H - 1);
        float penum = LoadR16F(a.penumbra, tx, ty);
        float zs = fabsf(LoadR32F(a.z, tx, ty) * c.gViewZScale);
        S s = shadowAt(tx, ty, penum);
        f2 uvs = mk2(__fmul_rn(__fadd_rn(fx, 0.5f), c.gRectSizeInv[0]), __fmul_rn(__fadd_rn(fy, 0.5f), c.gRectSizeInv[1]));
        f3 Xvs = ReconstructViewPosition(uvs, c.gFrustum, zs, c.gOrthoMode);
        float w = inScreen ? 1.0f : 0.0f;
        w *= NonExpWeight(dot(Nv, Xvs), geoA, geoB);
        w *= sg::BothLitOrUnlit(centerPenumbra, penum);
        w *= n < 4 ? 0.516851340f : 0.847893725f; // exp(-0.66 * r^2), r = 1 / 0.5
        w *= saturate(penum * invEstimatedPenumbra);
        if (w != 0.0f) result = result + sgt::Scale(s, w);
        sumX += w;
        w *= pixelSize / (pixelSize + penum);
        w *= sg::IsLit(penum) ? 0.0f : 1.0f;
        penumbra += w == 0.0f ? 0.0f : penum * w;
        sumY += w;
    }
    result = sgt::Scale(result, 1.0f / sumX);
    penumbra = sumY == 0.0f ? centerPenumbra : penumbra / sumY;

    if (FIRST || c.gStabilizationStrength != 0.0f) StoreR16F(a.outPenumbra, x, y, penumbra);
    sgt::Store(a.outShadow, x, y, sgt::Pack(result));
}

// ---------------------------------------------------------------------------------------------
struct SigmaTsArgs
{
    SigmaConstants c;
    Surf z, mv, penumbra, shadow, history, historyLength, tiles, outShadow, outLength;
    int rowBegin, rowEnd;
};

__device__ __forceinline__ unsigned PackViewZAndHistoryLength(float viewZ, float historyLength)
{
    return (__float_as_uint(viewZ) & ~7u) | min((unsigned)(historyLength + 0.5f), 7u);
}

template <class S> __device__ __forceinline__ S SigClamped(const Surf& s, int x, int y)
{
    S v;
    sgt::Load(s, clampi(x, 0, s.w - 1), clampi(y, 0, s.h - 1), v);
    return v;
}
template <class S> __device__ __forceinline__ S SampleLinearSig(const Surf& s, float u, float v)
{
    float px = u * (float)s.w - 0.5f, py = v * (float)s.h - 0.5f;
    float fx = floorf(px), fy = floorf(py), wx = px - fx, wy = py - fy;
    int x0 = (int)fx, y0 = (int)fy;
    return sgt::Lerp(sgt::Lerp(SigClamped<S>(s, x0, y0), SigClamped<S>(s, x0 + 1, y0), wx), sgt::Lerp(SigClamped<S>(s, x0, y0 + 1), SigClamped<S>(s, x0 + 1, y0 + 1), wx), wy);
}

template <bool TR>
__global__ void __launch_bounds__(256) SigmaTemporalStabilizationKernel(const __grid_constant__ SigmaTsArgs a)
{
    typedef typename sgt::Sig<TR>::T S;
    const SigmaConstants& c = a.c;
    const int x = blockIdx.x * 32 + threadIdx.x, y = a.rowBegin + blockIdx.y * 8 + threadIdx.y;
    const int maxX = c.gRectSizeMinusOne[0], maxY = c.gRectSizeMinusOne[1];
    if (x > maxX || y > maxY || y >= a.rowEnd) return;
    if (LoadRG8Unorm(a.tiles, x >> 4, y >> 4).x != 0.0f) return;
    const float viewZ = fabsf(LoadR32F(a.z, x, y) * c.gViewZScale);
    if (viewZ > c.gDenoisingRange) return;
    const float centerPenumbra = LoadR16F(a.penumbra, x, y);

    const f2 pixelUv = PixelUv(x, y, c.gRectSizeInv);
    const float tileValue = sg::TextureCubic(a.tiles, pixelUv.x * c.gResolutionScale[0], pixelUv.y * c.gResolutionScale[1]).y;
    if (tileValue == 0.0f || centerPenumbra == 0.0f)
    {
        S s;
        sgt::Load(a.shadow, x, y, s);
        sgt::Store(a.outShadow, x, y, sgt::Pack(sgt::Sq(s)));
        StoreU32(a.outLength, x, y, PackViewZAndHistoryLength(viewZ, 7.0f));
        return;
    }

    float sum = 0.0f;
    S m1 = sgt::Splat(0.0f, S()), m2 = sgt::Splat(0.0f, S()), input = sgt::Splat(0.0f, S());
#pragma unroll
    for (int j = -2; j <= 2; j++)
#pragma unroll
        for (int i = -2; i <= 2; i++)
        {
            int px = clampi(x + i, 0, maxX), py = clampi(y + j, 0, maxY);
            S s;
            sgt::Load(a.shadow, px, py, s);
            s = sgt::Sq(s);
            float w = 1.0f;
            if (i == 0 && j == 0) input = s;
            else
            {
                w = sg::BothLitOrUnlit(centerPenumbra, LoadR16F(a.penumbra, px, py));
                w *= __expf(-0.66f * (float)(i * i + j * j) * 0.25f);
            }
            m1 = m1 + sgt::Scale(s, w);
            m2 = m2 + sgt::Scale(sgt::Sq(s), w);
            sum += w;
        }
    m1 = sgt::Scale(m1, 1.0f / sum);
    m2 = sgt::Scale(m2, 1.0f / sum);
    S sigma = sgt::StdDev(m1, m2);

    const f3 Xv = ReconstructViewPosition(pixelUv, c.gFrustum, viewZ, c.gOrthoMode);
    const f3 X = PinnedRotateInverse(c.gWorldToView, Xv);
    const f4 mvRaw = LoadRGBA16F(a.mv, x, y);
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

    // bilinear footprint of the packed (viewZ | history length) texture
    float tx = __fadd_rn(__fmul_rn(smbPixelUv.x, c.gRectSizePrev[0]), -0.5f), ty = __fadd_rn(__fmul_rn(smbPixelUv.y, c.gRectSizePrev[1]), -0.5f);
    float ox = floorf(tx), oy = floorf(ty), wx = __fadd_rn(tx, -ox), wy = __fadd_rn(ty, -oy);
    int bx = (int)ox, by = (int)oy;
    const int W1 = a.historyLength.w - 1, H1 = a.historyLength.h - 1;
    unsigned d00 = LoadU32(a.historyLength, clampi(bx, 0, W1), clampi(by, 0, H1)), d10 = LoadU32(a.historyLength, clampi(bx + 1, 0, W1), clampi(by, 0, H1));
    unsigned d01 = LoadU32(a.historyLength, clampi(bx, 0, W1), clampi(by + 1, 0, H1)), d11 = LoadU32(a.historyLength, clampi(bx + 1, 0, W1), clampi(by + 1, 0, H1));

    const float frustumSize = c.gMinRectDimMulUnproject * lerpf(viewZ, 1.0f, fabsf(c.gOrthoMode));
    float thr = frustumSize * saturate(0.02f / fmaxf(0.01f, 1.0f));
    thr *= (smbPixelUv.x > 0.0f && smbPixelUv.y > 0.0f && smbPixelUv.x < 1.0f && smbPixelUv.y < 1.0f) ? 1.0f : 0.0f;
    thr -= kEps;
    const float XvprevZ = PinnedRow(c.gWorldToViewPrev, 2, Xprev.x, Xprev.y, Xprev.z);
    auto occ = [&](unsigned d) { return fabsf(__uint_as_float(d & ~7u) - XvprevZ) <= thr ? 1.0f : 0.0f; };
    float ooX = 1.0f - wx, ooY = 1.0f - wy;
    f4 w4 = mk4(occ(d00) * (ooX * ooY), occ(d10) * (wx * ooY), occ(d01) * (ooX * wy), occ(d11) * (wx * wy));
    float wsum = w4.x + w4.y + w4.z + w4.w;
    float hl = (float)(d00 & 7u) * w4.x + (float)(d10 & 7u) * w4.y + (float)(d01 & 7u) * w4.z + (float)(d11 & 7u) * w4.w;
    float historyLength = wsum < 0.0001f ? 0.0f : hl / wsum;

    // history: CatRom-12 when the whole footprint is valid, else custom-weight bilinear (through the bilinear sampler taps)
    const bool useBicubic = wsum > 3.5f;
    S history;
    {
        float spx = saturate(smbPixelUv.x) * c.gRectSizePrev[0], spy = saturate(smbPixelUv.y) * c.gRectSizePrev[1];
        float cx = floorf(spx - 0.5f) + 0.5f, cy = floorf(spy - 0.5f) + 0.5f;
        float fx = saturate(spx - cx), fy = saturate(spy - cy);
        const float kS = 0.5f; // CatRom sharpness
        float w0x = fx * (fx * (-kS * fx + 2.0f * kS) - kS), w0y = fy * (fy * (-kS * fy + 2.0f * kS) - kS);
        float w1x = fx * (fx * ((2.0f - kS) * fx - (3.0f - kS))) + 1.0f, w1y = fy * (fy * ((2.0f - kS) * fy - (3.0f - kS))) + 1.0f;
        float w2x = fx * (fx * (-(2.0f - kS) * fx + (3.0f - 2.0f * kS)) + kS), w2y = fy * (fy * (-(2.0f - kS) * fy + (3.0f - 2.0f * kS)) + kS);
        float w3x = fx * (fx * (kS * fx - kS)), w3y = fy * (fy * (kS * fy - kS));
        float w12x = w1x + w2x, w12y = w1y + w2y, tcx = w2x / w12x, tcy = w2y / w12y;
        f4 w = useBicubic ? mk4(w12x * w0y, w0x * w12y, w12x * w12y, w3x * w12y) : w4;
        float wl = useBicubic ? w12x * w3y : 0.0f;
        float total = w.x + w.y + w.z + w.w + wl;
        const float ix = c.gResourceSizeInvPrev[0], iy = c.gResourceSizeInvPrev[1];
        S col;
        if (useBicubic)
        {
            col = sgt::Scale(SampleLinearSig<S>(a.history, (cx + tcx) * ix, (cy - 1.0f) * iy), w.x);
            col = col + sgt::Scale(SampleLinearSig<S>(a.history, (cx - 1.0f) * ix, (cy + tcy) * iy), w.y);
            col = col + sgt::Scale(SampleLinearSig<S>(a.history, (cx + tcx) * ix, (cy + tcy) * iy), w.z);
            col = col + sgt::Scale(SampleLinearSig<S>(a.history, (cx + 2.0f) * ix, (cy + tcy) * iy), w.w);
            col = col + sgt::Scale(SampleLinearSig<S>(a.history, (cx + tcx) * ix, (cy + 2.0f) * iy), wl);
        }
        else
        {
            col = sgt::Scale(SampleLinearSig<S>(a.history, cx * ix, cy * iy), w.x);
            col = col + sgt::Scale(SampleLinearSig<S>(a.history, (cx + 1.0f) * ix, cy * iy), w.y);
            col = col + sgt::Scale(SampleLinearSig<S>(a.history, cx * ix, (cy + 1.0f) * iy), w.z);
            col = col + sgt::Scale(SampleLinearSig<S>(a.history, (cx + 1.0f) * ix, (cy + 1.0f) * iy), w.w);
        }
        history = total < 0.0001f ? sgt::Splat(0.0f, S()) : sgt::Scale(col, 1.0f / total);
    }
    history = sgt::Sq(sgt::Sat(history));

    sigma = sgt::Scale(sigma, lerpf(3.0f, 1.0f, 1.0f / (1.0f + historyLength)));
    S historyClamped = sgt::Clamp(history, m1 - sigma, m1 + sigma);
    float antilag = saturate(1.0f - Sqrt01(fabsf(sgt::X(historyClamped) - sgt::X(history)))); // ".x" only (SIGMA_TemporalStabilization.hlsli:174)
    historyLength *= antilag;
    float historyWeight = historyLength / (1.0f + historyLength);
    historyClamped = sgt::Lerp(historyClamped, history, 0.6f * historyWeight * antilag);
    S result = sgt::Lerp(input, historyClamped, fminf(c.gStabilizationStrength, historyWeight));
    historyLength = fminf(historyLength + 1.0f, 7.0f);

    sgt::Store(a.outShadow, x, y, sgt::Pack(result));
    StoreU32(a.outLength, x, y, PackViewZAndHistoryLength(viewZ, historyLength));
}

// ---------------------------------------------------------------------------------------------
cudaError_t LaunchSigma(const PassLaunch& p)
{
    const SigmaConstants& c = *(const SigmaConstants*)p.constants;
    const int W = (int)c.gRectSize[0];
    // SIGMA_TYPE float (SIGMA_Shadow_*) or float4 (SIGMA_ShadowTranslucency_*); SmoothTiles and Copy are shared, Copy sees which one
    // it serves from the format of the history texture (p.texBytes)
    const bool translucent = p.kind.translucent;
    Bindings b(p);
    if (p.kind.pass == Pass::ClassifyTiles)
    {
        SigmaTilesArgs a;
        a.z = b.Next(); a.penumbra = b.Next(); a.translucency = b.Next(translucent); a.tiles = b.Next();
        if (!b.Complete()) return cudaErrorInvalidValue;
        a.viewZScale = c.gViewZScale; a.denoisingRange = c.gDenoisingRange; a.unproject = c.gUnproject; a.orthoMode = c.gOrthoMode;
        a.tilesW = p.gridW; a.tilesH = p.gridH;
        int warps = a.tilesW * a.tilesH;
        if (translucent) NRD_B200_LAUNCH(p, (warps * 32 + 255) / 256, 256, a, SigmaClassifyTilesKernel<true>);
        else NRD_B200_LAUNCH(p, (warps * 32 + 255) / 256, 256, a, SigmaClassifyTilesKernel<false>);
    }
    else if (p.kind.pass == Pass::SmoothTiles)
    {
        SigmaSmoothArgs a;
        a.tiles = b.Next(); a.smoothed = b.Next();
        if (!b.Complete()) return cudaErrorInvalidValue;
        a.tilesMaxX = c.gTilesSizeMinusOne[0]; a.tilesMaxY = c.gTilesSizeMinusOne[1];
        NRD_B200_LAUNCH(p, dim3(p.gridW, p.gridH), dim3(16, 16), a, SigmaSmoothTilesKernel);
    }
    else if (p.kind.pass == Pass::Copy)
    {
        SigmaCopyArgs a;
        a.tiles = b.Next(); a.inHistory = b.Next(); a.inLength = b.Next(); a.outHistory = b.Next(); a.outLength = b.Next();
        if (!b.Complete()) return cudaErrorInvalidValue;
        a.w = a.inHistory.w; a.h = a.inHistory.h; a.isRectChanged = c.gIsRectChanged; a.rowBegin = p.rowBegin; a.rowEnd = p.rowEnd;
        const dim3 grid((a.w + 31) / 32, (p.rowEnd - p.rowBegin + 7) / 8), block(32, 8);
        if (p.preloadOnly || p.texBytes[3] == 4) NRD_B200_LAUNCH(p, grid, block, a, SigmaCopyKernel<true>);
        if (p.preloadOnly || p.texBytes[3] != 4) NRD_B200_LAUNCH(p, grid, block, a, SigmaCopyKernel<false>);
    }
    else if (p.kind.pass == Pass::Blur || p.kind.pass == Pass::PostBlur)
    {
        const bool first = p.kind.pass == Pass::Blur;
        SigmaBlurArgs a;
        a.c = c;
        a.z = b.Next(); a.nr = b.Next(); a.penumbra = b.Next(); a.tiles = b.Next();
        a.shadow = b.Next(!first || translucent); // SIGMA_Blur.resources.hlsli:25-27
        a.outPenumbra = b.Next(); a.outShadow = b.Next();
        if (!b.Complete()) return cudaErrorInvalidValue;
        a.rowBegin = p.rowBegin; a.rowEnd = p.rowEnd;
        dim3 grid((W + 31) / 32, (p.rowEnd - p.rowBegin + 7) / 8), block(32, 8);
        if (first && translucent) NRD_B200_LAUNCH(p, grid, block, a, SigmaBlurKernel<true, true>);
        else if (first) NRD_B200_LAUNCH(p, grid, block, a, SigmaBlurKernel<true, false>);
        else if (translucent) NRD_B200_LAUNCH(p, grid, block, a, SigmaBlurKernel<false, true>);
        else NRD_B200_LAUNCH(p, grid, block, a, SigmaBlurKernel<false, false>);
    }
    else if (p.kind.pass == Pass::TemporalStabilization)
    {
        SigmaTsArgs a;
        a.c = c;
        a.z = b.Next(); a.mv = b.Next(); a.penumbra = b.Next(); a.shadow = b.Next(); a.history = b.Next(); a.historyLength = b.Next(); a.tiles = b.Next();
        a.outShadow = b.Next(); a.outLength = b.Next();
        if (!b.Complete()) return cudaErrorInvalidValue;
        a.rowBegin = p.rowBegin; a.rowEnd = p.rowEnd;
        const dim3 grid((W + 31) / 32, (p.rowEnd - p.rowBegin + 7) / 8), block(32, 8);
        if (translucent) NRD_B200_LAUNCH(p, grid, block, a, SigmaTemporalStabilizationKernel<true>);
        else NRD_B200_LAUNCH(p, grid, block, a, SigmaTemporalStabilizationKernel<false>);
    }
    else
        return cudaErrorNotSupported;
    return cudaGetLastError();
}

#if !defined(NRD_B200_NO_STRIPS)
cudaError_t SetPeerTableSigma(int slot, const PeerTable* table, const cudaStream_t* stream) { return SetPeerTableThisTU(slot, table, stream); }
#endif
} // namespace nrdb200
