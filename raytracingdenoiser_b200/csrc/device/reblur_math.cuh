// REBLUR per-pixel math for the sm_90a kernels (device functions only).
// What each function has to compute is defined by the reference shaders (cited per function); how it is computed here is
// organised for the GPU: guides are decoded once, uniform work is hoisted, transcendental-heavy parameters are per pixel
// not per tap, and texel-selecting arithmetic is pinned (see common.cuh).
#pragma once
#include "common.cuh" // first: selects the namespace of this build of the kernels
#include "../constants.h"

namespace nrdb200
{
namespace rb
{
constexpr float kEps = 1e-6f;                         // NRD_EPS            NRD.hlsli:313
constexpr float kInf = 1e6f;                          // NRD_INF            NRD.hlsli:316
constexpr float kNormalEncodingError = 0.75f / 255.0f; // Common.hlsli:79-81 (R10G10B10A2)
constexpr float kMaxAccum = 63.0f;                    // REBLUR_MAX_ACCUM_FRAME_NUM
constexpr float kMaxMaterial = 15.0f;                 // REBLUR_MAX_MATERIALID_NUM
constexpr float kLobeVolume = 0.75f;                  // NRD_MAX_PERCENT_OF_LOBE_VOLUME

// ---- guides -------------------------------------------------------------------------------------
// NRD_FrontEnd_UnpackNormalAndRoughness for R10G10B10A2 / linear roughness (NRD.hlsli:600-628, 337-347, 321-324)
struct Guide
{
    f3 N;
    float roughness;
    float materialID;
    float smc, hitK, aLog; // roughness-table entry (LoadGuideLut): SpecMagicCurve, hit-distance normalisation factor, dominant-direction log term
};
__device__ __forceinline__ Guide DecodeGuide(unsigned packed)
{
    float px = (float)(packed & 1023u) / 1023.0f, py = (float)((packed >> 10) & 1023u) / 1023.0f;
    float nx = px * 2.0f - 1.0f, ny = py * 2.0f - 1.0f;
    float nz = 1.0f - fabsf(nx) - fabsf(ny);
    float t = saturate(-nz);
    nx -= t * (nx >= 0.0f ? 1.0f : -1.0f);
    ny -= t * (ny >= 0.0f ? 1.0f : -1.0f);
    float inv = rsqrtf(nx * nx + ny * ny + nz * nz + 1e-9f);
    Guide g;
    g.N = mk3(nx * inv, ny * inv, nz * inv);
    g.roughness = (float)((packed >> 20) & 1023u) / 1023.0f;
    g.materialID = ((float)(packed >> 30) / 3.0f) * 3.0f;
    return g;
}

// NRD_FrontEnd_UnpackNormalAndRoughness (NRD.hlsli:600-628, R10G10B10A2) in the oracle's operation order with IEEE division and
// square root: the stored normal is bit-identical to the oracle's.  Once per pixel and frame, so the ~20 extra instructions are free.
__device__ __forceinline__ f3 DecodeNormalExact(unsigned packed)
{
    const float px = __fdiv_rn((float)(packed & 1023u), 1023.0f), py = __fdiv_rn((float)((packed >> 10) & 1023u), 1023.0f);
    float nx = __fadd_rn(__fmul_rn(px, 2.0f), -1.0f), ny = __fadd_rn(__fmul_rn(py, 2.0f), -1.0f);
    const float nz = __fadd_rn(__fadd_rn(1.0f, -fabsf(nx)), -fabsf(ny));
    const float t = saturate(-nz);
    nx = __fadd_rn(nx, nx >= 0.0f ? -t : t);
    ny = __fadd_rn(ny, ny >= 0.0f ? -t : t);
    const float d = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(nx, nx), __fmul_rn(ny, ny)), __fmul_rn(nz, nz)), 1e-9f);
    const float inv = __fdiv_rn(1.0f, __fsqrt_rn(d));
    return mk3(__fmul_rn(nx, inv), __fmul_rn(ny, inv), __fmul_rn(nz, inv));
}

// Guides through the decoded-guide surface (surf.h PassLaunch::guide: {N.xyz bit-exact, |viewZ * gViewZScale| for REBLUR, raw viewZ for RELAX}, written by ClassifyTiles at
// the start of every frame): one 16-byte load instead of the octahedral decode; roughness / material straight from the packed
// bits (loads whose result is unused are removed by the compiler).
__device__ __forceinline__ Guide LoadGuide(const Surf& guide, const Surf& nr, int x, int y)
{
    const f4 q = LoadRGBA32F(guide, x, y);
    const unsigned p = LoadU32(nr, x, y);
    Guide g;
    g.N = mk3(q.x, q.y, q.z);
    g.roughness = (float)((p >> 20) & 1023u) * (1.0f / 1023.0f);
    g.materialID = (float)(p >> 30);
    return g;
}

// ... plus everything that depends on the 10-bit roughness alone, from the host-built table (surf.h PassLaunch::roughnessLut):
// no powf / exp2f / logf in the kernel, and the values are the oracle's bit for bit
__device__ __forceinline__ Guide LoadGuideLut(const Surf& guide, const Surf& nr, const float4* lut, int x, int y)
{
    const f4 q = LoadRGBA32F(guide, x, y);
    const unsigned p = LoadU32(nr, x, y);
    const float4 t = __ldg(&lut[(p >> 20) & 1023u]);
    Guide g;
    g.N = mk3(q.x, q.y, q.z);
    g.roughness = t.w; // exactly i / 1023
    g.materialID = (float)(p >> 30);
    g.smc = t.x;
    g.hitK = t.y;
    g.aLog = t.z;
    return g;
}

// ---- scalar helpers -----------------------------------------------------------------------------
__device__ __forceinline__ float SmoothStep01(float x) { float t = saturate(x); return t * t * (3.0f - 2.0f * t); }
__device__ __forceinline__ float LinearStep(float a, float b, float x) { return SatMul(x - a, __fdividef(1.0f, b - a)); }
__device__ __forceinline__ float SmoothStep(float a, float b, float x) { return SmoothStep01(LinearStep(a, b, x)); }
__device__ __forceinline__ float Sqrt01(float x) { return sqrtf(saturate(x)); }
__device__ __forceinline__ float Pow01(float x, float y) { return powf(saturate(x), y); }
__device__ __forceinline__ float PositiveRcp(float x) { return 1.0f / fmaxf(x, 1e-15f); }
__device__ __forceinline__ float AcosApprox(float x) { return 1.41421356f * sqrtf(OneMinusSat(x)); }
__device__ __forceinline__ float Pow5(float x) { float t = OneMinusSat(x); float t2 = t * t; return t2 * t2 * t; } // pow(saturate(1-x),5)
__device__ __forceinline__ float GetStdDev(float m1, float m2) { return sqrtf(fabsf(m2 - m1 * m1)); }
// floor(x) for |x| < 2^22 without the conversion pipe: x + 1.5 * 2^23 rounded towards -inf has floor(x) in its low mantissa bits.
// Anything outside that range (inf, NaN, a tap projected from behind the camera) comes out as an index far outside any screen.
__device__ __forceinline__ float FloorIndex(float x, int& i)
{
    const float t = __fadd_rd(x, 12582912.0f);
    i = __float_as_int(t) - 0x4B400000;
    return __fadd_rn(t, -12582912.0f);
}

// Sequence::CheckerBoard (REBLUR_PrePass.hlsli:44): which half of the pixels carries data this frame
__device__ __forceinline__ unsigned CheckerBoard(int x, int y, unsigned frameIndex) { return (((unsigned)x ^ (unsigned)y) ^ frameIndex) & 1u; }
// Sequence::Bayer4x4 (frozen: standard 4x4 ordered-dither matrix, see oracle/mathlib.h).  The templates are a codegen pin, not
// part of the dither: they keep the table out of the units that never call Bayer4x4, because with nvcc 12.9 a table in constant
// bank 3 moves the strip build's peer table (common.cuh) and changes the code of every strip-build kernel of the unit.
// Revisit with the next nvcc.
template <class T = unsigned> static __constant__ T kBayer4x4[16] = {0, 8, 2, 10, 12, 4, 14, 6, 3, 11, 1, 9, 15, 7, 13, 5};
template <class T = unsigned> __device__ __forceinline__ float Bayer4x4(int x, int y, unsigned frameIndex)
{
    return (float)((kBayer4x4<T>[(y & 3) * 4 + (x & 3)] + frameIndex) & 15u) / 16.0f;
}

// weights: Common.hlsli:547-574 (SmoothStep(1,0,x) == smoothstep01(1 - x))
__device__ __forceinline__ float NonExpWeight(float x, float px, float py)
{
    const float u = OneMinusAbsSat(fmaf(x, px, py));
    return u * u * fmaf(-2.0f, u, 3.0f);
}
__device__ __forceinline__ float NonExpWeightWithSigma(float x, float px, float py, float sigma) { return SmoothStep01(1.0f - (fabsf(x * px + py) - sigma * px)); }
__device__ __forceinline__ float ExpWeight(float x, float px, float py)
{
    float v = -3.0f * fabsf(x * px + py);
    return __fdividef(1.0f, v * v - v + 1.0f); // a weight in (0, 1]: the 2-ulp reciprocal is enough (the IEEE one costs ~8 instructions per tap)
}
__device__ __forceinline__ float EncodingAwareNormalWeight(f3 Ncurr, f3 Nprev, float maxAngle, float curvatureAngle, float thresholdAngle, bool remap = false) // Common.hlsli:578-590
{
    float angle = AcosApprox(dot(Ncurr, Nprev));
    float w = SmoothStep01(1.0f - (angle - curvatureAngle - thresholdAngle) / maxAngle);
    return remap ? SmoothStep(0.05f, 0.95f, w) : w;
}

__device__ __forceinline__ float HitDistNormalization(float viewZ, const float* p, float roughness) // NRD.hlsli:520-523
{
    return (p[0] + fabsf(viewZ) * p[1]) * lerpf(1.0f, p[2], saturate(exp2f(p[3] * roughness * roughness)));
}
__device__ __forceinline__ float SpecMagicCurve(float roughness) // Common.hlsli:311-317, power = 0.25: the fourth root as two square roots
{
    float f = 1.0f - exp2f(-200.0f * roughness * roughness);
    return f * sqrtf(sqrtf(saturate(roughness)));
}
// Filtering::GetModifiedRoughnessFromNormalVariance (restated in oracle/mathlib.h): avgN is the non-normalised average normal
__device__ __forceinline__ float ModifiedRoughness(float roughness, f3 avgN)
{
    float l = length(avgN);
    float kappa = saturate(1.0f - l * l) / fmaxf(l * (3.0f - l * l), 1e-15f);
    return Sqrt01(roughness * roughness + kappa);
}
__device__ __forceinline__ float LobeTanHalfAngle(float roughness, float percentOfVolume) // MathLib ImportanceSampling (restated, see oracle/mathlib.h)
{
    float m = saturate(roughness);
    m *= m;
    return m * sqrtf(percentOfVolume / (1.0f - percentOfVolume + 1e-6f));
}
__device__ __forceinline__ float NormalWeightParam(float nonLinearAccumSpeed, float lobeAngleFraction, float roughness) // Common.hlsli:486-500
{
    float percentOfVolume = kLobeVolume * lerpf(lobeAngleFraction, 1.0f, nonLinearAccumSpeed);
    float angle = atanf(LobeTanHalfAngle(roughness, percentOfVolume));
    return 1.0f / fmaxf(angle, kNormalEncodingError);
}
__device__ __forceinline__ f2 HitDistanceWeightParams(float hitDist, float nonLinearAccumSpeed, float smc) // Common.hlsli:511-522 (smc = SpecMagicCurve(roughness))
{
    float a = 1.0f / lerpf(0.0005f, 1.0f, fminf(nonLinearAccumSpeed, smc));
    return mk2(a, -hitDist * a);
}
__device__ __forceinline__ f2 RoughnessWeightParams(float roughness, float fraction, float sensitivity = 0.01f) // Common.hlsli:524-530
{
    float a = 1.0f / lerpf(sensitivity, 1.0f, saturate(roughness * fraction));
    return mk2(a, -roughness * a);
}
__device__ __forceinline__ f2 RelaxedRoughnessWeightParams(float m, float fraction, float sensitivity = 0.01f) // Common.hlsli:532-541
{
    float a = 1.0f / lerpf(sensitivity, 1.0f, lerpf(m * m, m, fraction));
    return mk2(a, -m * a);
}
__device__ __forceinline__ float SpecularDominantFactor(float NoV, float roughness) // NRD.hlsli:386-392
{
    float a = 0.298475f * logf(39.4115f - 39.0029f * roughness);
    return saturate(powf(saturate(1.0f - NoV), 10.8649f) * (1.0f - a) + a);
}
// the same with the roughness-only log term a = 0.298475 log(39.4115 - 39.0029 r) taken from the roughness table
__device__ __forceinline__ float SpecularDominantFactorLut(float NoV, float aLog) { return SatFma(powf(OneMinusSat(NoV), 10.8649f), 1.0f - aLog, aLog); }
__device__ __forceinline__ f4 SpecularDominantDirectionLut(f3 N, f3 V, float aLog)
{
    const float f = SpecularDominantFactorLut(fabsf(dot(N, V)), aLog);
    return mk4(normalize(lerp3(N, reflect(-V, N), f)), f);
}
__device__ __forceinline__ f4 SpecularDominantDirection(f3 N, f3 V, float roughness) // NRD.hlsli:394-400
{
    float f = SpecularDominantFactor(fabsf(dot(N, V)), roughness);
    f3 R = reflect(-V, N);
    return mk4(normalize(lerp3(N, R, f)), f);
}
// branchless orthonormal basis, rows T, B (MathLib Geometry::GetBasis restated)
__device__ __forceinline__ void GetBasis(f3 N, f3& T, f3& B)
{
    float sz = N.z < 0.0f ? -1.0f : 1.0f;
    float a = 1.0f / (sz + N.z);
    float ya = N.y * a;
    float b = N.x * ya;
    float c = N.x * sz;
    T = mk3(c * N.x * a - 1.0f, sz * b, c);
    B = mk3(b, N.y * ya - sz, N.y);
}
__device__ __forceinline__ void KernelBasis(f3 D, f3 N, f3& T, f3& B) // REBLUR_Common.hlsli:278-293
{
    GetBasis(N, T, B);
    if (fabsf(dot(D, N)) < 0.999f)
    {
        f3 R = reflect(-D, N);
        T = normalize(cross(N, R));
        B = cross(R, T);
    }
}

// colour helpers (YCoCg signals): REBLUR_Common.hlsli:139-146, 211-240; NRD.hlsli:356-375
__device__ __forceinline__ float LumaScale(float cur, float nw) { return (nw + kEps) / (cur + kEps); }
__device__ __forceinline__ f4 ChangeLuma(f4 v, float newLuma)
{
    float s = LumaScale(v.x, newLuma);
    return mk4(v.x * s, v.y * s, v.z * s, v.w);
}
__device__ __forceinline__ f4 ClampNegativeToZero(f4 v)
{
    float t = v.x - v.z;
    float g = fmaxf(v.x + v.z, 0.0f), r = fmaxf(t + v.y, 0.0f), b = fmaxf(t - v.y, 0.0f);
    f4 o;
    o.x = r * 0.25f + g * 0.5f + b * 0.25f;
    o.y = r * 0.5f + g * 0.0f + b * -0.5f;
    o.z = r * -0.25f + g * 0.5f + b * -0.25f;
    o.w = saturate(v.w);
    return o;
}

// packed records: REBLUR_Common.hlsli:13-80
__device__ __forceinline__ unsigned PackInternalData(float diffAccum, float specAccum, float materialID)
{
    unsigned p = ToUnorm(__fdiv_rn(diffAccum, kMaxAccum), 63.0f);
    p |= ToUnorm(__fdiv_rn(specAccum, kMaxAccum), 63.0f) << 6;
    p |= ToUnorm(__fdiv_rn(materialID, kMaxMaterial), 15.0f) << 12;
    return p;
}
__device__ __forceinline__ f3 UnpackInternalData(unsigned p)
{
    // (n / 63) * 63 and (n / 15) * 15 of the reference are n up to one rounding: no divisions
    return mk3((float)(p & 63u), (float)((p >> 6) & 63u), (float)((p >> 12) & 15u));
}
__device__ __forceinline__ unsigned PackData2(float fbits, float curvature, float virtualHistoryAmount)
{
    unsigned p = (unsigned)(fbits + 0.5f);
    p |= ToUnorm(virtualHistoryAmount, 255.0f) << 8;
    p |= (unsigned)__half_as_ushort(__float2half_rn(curvature)) << 16;
    return p;
}

// ---- pinned geometry ----------------------------------------------------------------------------
// pixelUv = (pixelPos + 0.5) * rectSizeInv
__device__ __forceinline__ f2 PixelUv(int x, int y, const float* rectSizeInv)
{
    return mk2(__fmul_rn(__fadd_rn((float)x, 0.5f), rectSizeInv[0]), __fmul_rn(__fadd_rn((float)y, 0.5f), rectSizeInv[1]));
}
// Geometry::ReconstructViewPosition (restated in oracle/mathlib.h): p.xy = (uv * frustum.zw + frustum.xy) * (viewZ * (1 - |ortho|) + ortho)
__device__ __forceinline__ f3 ReconstructViewPosition(f2 uv, const float* frustum, float viewZ, float orthoMode)
{
    float scale = __fadd_rn(__fmul_rn(viewZ, __fadd_rn(1.0f, -fabsf(orthoMode))), orthoMode);
    float x = __fmul_rn(__fadd_rn(__fmul_rn(uv.x, frustum[2]), frustum[0]), scale);
    float y = __fmul_rn(__fadd_rn(__fmul_rn(uv.y, frustum[3]), frustum[1]), scale);
    return mk3(x, y, viewZ);
}
// Geometry::GetScreenUv: uv = clip.xy / clip.w * (0.5, -0.5) + 0.5, uv = 99999 behind the camera
__device__ __forceinline__ f2 GetScreenUv(const float* m, f3 X)
{
    float cx = PinnedRow(m, 0, X.x, X.y, X.z), cy = PinnedRow(m, 1, X.x, X.y, X.z), cw = PinnedRow(m, 3, X.x, X.y, X.z);
    f2 uv = mk2(__fadd_rn(__fmul_rn(__fdiv_rn(cx, cw), 0.5f), 0.5f), __fadd_rn(__fmul_rn(__fdiv_rn(cy, cw), -0.5f), 0.5f));
    if (cw < 0.0f) uv = mk2(99999.0f, 99999.0f);
    return uv;
}
__device__ __forceinline__ f3 AffineTransform(const float* m, f3 X)
{
    return mk3(PinnedRow(m, 0, X.x, X.y, X.z), PinnedRow(m, 1, X.x, X.y, X.z), PinnedRow(m, 2, X.x, X.y, X.z));
}
} // namespace rb
} // namespace nrdb200
