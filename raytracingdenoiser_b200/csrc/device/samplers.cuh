// Software samplers with D3D clamp-to-edge addressing and the CatRom-12 / custom-weight bilinear history filter
// (Common.hlsli:602-656), shared by the REBLUR and RELAX temporal passes.
// In the strip build, with FOOTPRINT_TEST (REBLUR) each footprint takes one FootprintLocal() test and is read through Near()
// views when all its rows are held locally (common.cuh); without it (RELAX) every load does the owner lookup.  The two forms
// compute the same sums, but ptxas fuses their multiplies and adds differently, so the form decides the strip build's output
// bytes: RELAX keeps the per-load form and with it the bytes it has always produced.
#pragma once
#include "common.cuh"

namespace nrdb200
{
__device__ __forceinline__ f4 FetchClamped4(const Surf& s, int x, int y) { return LoadRGBA16F(s, clampi(x, 0, s.w - 1), clampi(y, 0, s.h - 1)); }
__device__ __forceinline__ float FetchClamped1(const Surf& s, int x, int y) { return LoadR16F(s, clampi(x, 0, s.w - 1), clampi(y, 0, s.h - 1)); }

// rows [ya, yb] after clamping to the texture are local: the footprint can be read through Near(s) (common.cuh)
__device__ __forceinline__ bool FootprintLocal(const Surf& s, int ya, int yb) { return RowsLocal(s, clampi(ya, 0, s.h - 1), clampi(yb, 0, s.h - 1)); }

__device__ __forceinline__ float SampleLinear1Impl(const Surf& s, int x0, int y0, float wx, float wy)
{
    float a = lerpf(FetchClamped1(s, x0, y0), FetchClamped1(s, x0 + 1, y0), wx);
    float b = lerpf(FetchClamped1(s, x0, y0 + 1), FetchClamped1(s, x0 + 1, y0 + 1), wx);
    return lerpf(a, b, wy);
}
template <bool FOOTPRINT_TEST = true> __device__ __forceinline__ float SampleLinear1(const Surf& s, float u, float v)
{
    float px = u * (float)s.w - 0.5f, py = v * (float)s.h - 0.5f;
    float fx = floorf(px), fy = floorf(py);
    float wx = px - fx, wy = py - fy;
    int x0 = (int)fx, y0 = (int)fy;
    return FOOTPRINT_TEST && FootprintLocal(s, y0, y0 + 1) ? SampleLinear1Impl(Near(s), x0, y0, wx, wy) : SampleLinear1Impl(s, x0, y0, wx, wy);
}

// CatRom-12 (no corners) with fallback to the custom-weight bilinear footprint (Common.hlsli:602-656)
struct CatRomSetup
{
    // uv of the reference's five bilinear taps.  Nothing reads them: a codegen pin, not part of the filter.  Without them
    // nvcc 12.9 allocates the registers of the REBLUR temporal kernels differently; revisit with the next nvcc.
    float u01x, u01y, u01z, u01w, u23x, u23y, u23z, u23w, u4x, u4y;
    f4 w;
    float w4, sum;
    int bx, by;
    float tcx, tcy; // position of the merged inner taps between texel bx and bx+1 (by and by+1)
    bool bicubic;
};
__device__ __forceinline__ CatRomSetup SetupCatRom(f2 samplePos, const float* invSize, f4 customWeights, bool useBicubic)
{
    CatRomSetup s;
    // texel of the footprint's centre: floor, not a conversion to int, which rounds -0.5 (a sample within half a texel of the
    // top or left edge) towards texel 0 instead of -1; the reference's sampler taps are placed at centerPos itself
    const float x0 = floorf(samplePos.x - 0.5f), y0 = floorf(samplePos.y - 0.5f);
    float cx = x0 + 0.5f, cy = y0 + 0.5f;
    float fx = saturate(samplePos.x - cx), fy = saturate(samplePos.y - cy);
    const float S = 0.5f;
    float w0x = fx * (fx * (-S * fx + 2.0f * S) - S), w0y = fy * (fy * (-S * fy + 2.0f * S) - S);
    float w1x = fx * (fx * ((2.0f - S) * fx - (3.0f - S))) + 1.0f, w1y = fy * (fy * ((2.0f - S) * fy - (3.0f - S))) + 1.0f;
    float w2x = fx * (fx * (-(2.0f - S) * fx + (3.0f - 2.0f * S)) + S), w2y = fy * (fy * (-(2.0f - S) * fy + (3.0f - 2.0f * S)) + S);
    float w3x = fx * (fx * (S * fx - S)), w3y = fy * (fy * (S * fy - S));
    float w12x = w1x + w2x, w12y = w1y + w2y;
    float tcx = w2x / w12x, tcy = w2y / w12y;
    f4 w = mk4(w12x * w0y, w0x * w12y, w12x * w12y, w3x * w12y);
    float w4 = w12x * w3y;
    s.w = useBicubic ? w : customWeights;
    s.w4 = useBicubic ? w4 : 0.0f;
    s.sum = s.w.x + s.w.y + s.w.z + s.w.w + s.w4;
    if (useBicubic)
    {
        s.u01x = cx + tcx; s.u01y = cy - 1.0f; s.u01z = cx - 1.0f; s.u01w = cy + tcy;
        s.u23x = cx + tcx; s.u23y = cy + tcy;  s.u23z = cx + 2.0f; s.u23w = cy + tcy;
        s.u4x = cx + tcx;  s.u4y = cy + 2.0f;
    }
    else
    {
        s.u01x = cx;        s.u01y = cy;        s.u01z = cx + 1.0f; s.u01w = cy;
        s.u23x = cx;        s.u23y = cy + 1.0f; s.u23z = cx + 1.0f; s.u23w = cy + 1.0f;
        s.u4x = cx + fx;    s.u4y = cy + fy;
    }
    s.u01x *= invSize[0]; s.u01y *= invSize[1]; s.u01z *= invSize[0]; s.u01w *= invSize[1];
    s.u23x *= invSize[0]; s.u23y *= invSize[1]; s.u23z *= invSize[0]; s.u23w *= invSize[1];
    s.u4x *= invSize[0];  s.u4y *= invSize[1];
    s.bx = (int)x0;
    s.by = (int)y0;
    s.tcx = tcx;
    s.tcy = tcy;
    s.bicubic = useBicubic;
    return s;
}
// The reference takes 5 hardware-bilinear taps; a software bilinear tap is 4 loads + 3 lerps, i.e. 20 loads for a
// footprint of 12 distinct texels.  Here every texel is loaded once and weighted with (tap weight) x (its bilinear weight):
// the same polynomial, summed in a different order (differences ~1e-6 relative, far inside the parity tolerance).
// Without a valid bicubic footprint the filter degenerates to the 2x2 texels with the custom bilinear weights.
template <class LOAD> __device__ __forceinline__ auto ResolveCatRomTexels(const CatRomSetup& s, const Surf& tex, LOAD load) -> decltype(load(tex, 0, 0))
{
    typedef decltype(load(tex, 0, 0)) V;
    const int x0 = s.bx, y0 = s.by;
    V color;
    if (s.bicubic)
    {
        const float ax = 1.0f - s.tcx, bx = s.tcx, ay = 1.0f - s.tcy, by = s.tcy;
        color = load(tex, x0, y0 - 1) * (s.w.x * ax) + load(tex, x0 + 1, y0 - 1) * (s.w.x * bx);
        color = color + load(tex, x0 - 1, y0) * (s.w.y * ay) + load(tex, x0 - 1, y0 + 1) * (s.w.y * by);
        color = color + load(tex, x0, y0) * (s.w.z * ax * ay) + load(tex, x0 + 1, y0) * (s.w.z * bx * ay);
        color = color + load(tex, x0, y0 + 1) * (s.w.z * ax * by) + load(tex, x0 + 1, y0 + 1) * (s.w.z * bx * by);
        color = color + load(tex, x0 + 2, y0) * (s.w.w * ay) + load(tex, x0 + 2, y0 + 1) * (s.w.w * by);
        color = color + load(tex, x0, y0 + 2) * (s.w4 * ax) + load(tex, x0 + 1, y0 + 2) * (s.w4 * bx);
    }
    else
        color = load(tex, x0, y0) * s.w.x + load(tex, x0 + 1, y0) * s.w.y + load(tex, x0, y0 + 1) * s.w.z + load(tex, x0 + 1, y0 + 1) * s.w.w;
    return color;
}
template <bool FOOTPRINT_TEST = true> __device__ __forceinline__ f4 ResolveCatRom4(const CatRomSetup& s, const Surf& tex)
{
    auto load = [](const Surf& t, int x, int y) { return FetchClamped4(t, x, y); };
    f4 color = FOOTPRINT_TEST && FootprintLocal(tex, s.by - 1, s.by + 2) ? ResolveCatRomTexels(s, Near(tex), load) : ResolveCatRomTexels(s, tex, load);
    return s.sum < 0.0001f ? mk4(0.0f) : color * (1.0f / s.sum);
}
__device__ __forceinline__ float ResolveCatRom1(const CatRomSetup& s, const Surf& tex)
{
    auto load = [](const Surf& t, int x, int y) { return FetchClamped1(t, x, y); };
    float color = FootprintLocal(tex, s.by - 1, s.by + 2) ? ResolveCatRomTexels(s, Near(tex), load) : ResolveCatRomTexels(s, tex, load);
    return s.sum < 0.0001f ? 0.0f : color / s.sum;
}
// tex.Load(origin + offset) * customWeights, out-of-bounds loads return 0
__device__ __forceinline__ float LoadOrZero1(const Surf& s, int x, int y) { return Inside(s, x, y) ? LoadR16F(s, x, y) : 0.0f; }
__device__ __forceinline__ float BilinearCustom1Sum(const Surf& tex, int bx, int by, f4 cw)
{
    return LoadOrZero1(tex, bx, by) * cw.x + LoadOrZero1(tex, bx + 1, by) * cw.y + LoadOrZero1(tex, bx, by + 1) * cw.z + LoadOrZero1(tex, bx + 1, by + 1) * cw.w;
}
__device__ __forceinline__ float ResolveBilinearCustom1(const CatRomSetup& s, const Surf& tex, f4 cw)
{
    // the reference loads these four texels at int2(centerPos), a conversion that rounds towards zero: a footprint that starts
    // left of or above texel 0 is loaded one texel later than the CatRom footprint (Common.hlsli:648-656)
    const int bx = s.bx < 0 ? s.bx + 1 : s.bx, by = s.by < 0 ? s.by + 1 : s.by;
    float v = FootprintLocal(tex, by, by + 1) ? BilinearCustom1Sum(Near(tex), bx, by, cw) : BilinearCustom1Sum(tex, bx, by, cw);
    float sum = cw.x + cw.y + cw.z + cw.w;
    return sum < 0.0001f ? 0.0f : v / sum;
}
} // namespace nrdb200
