// RELAX_DIFFUSE_SPECULAR passes for sm_90a: classify tiles, pre-pass, temporal accumulation, history fix, history clamping
// (anti-lag), A-trous with the spatial-variance first iteration, A-trous.
// Behaviour follows the reference's shaders (cited per kernel); arithmetic that selects a texel / footprint or that is stored
// quantised is pinned to the oracle's operation order (oracle/relax.cpp), everything else is free to contract.
#include "launch.h" // first: selects the namespace of this build of the kernels
#include "../constants.h"
#include "reblur_math.cuh"
#include "samplers.cuh"

#include <cstring>

namespace nrdb200
{
namespace
{
using namespace rb;

constexpr float kNormalUlp = 1.5f / 255.0f;  // RELAX_NORMAL_ULP             RELAX_Config.hlsli
constexpr float kMaxAccumRelax = 255.0f;     // RELAX_MAX_ACCUM_FRAME_NUM
constexpr float kAntilagAccelScale = 10.0f;  // RELAX_ANTILAG_ACCELERATION_AMOUNT_SCALE
constexpr float kCurvatureZThreshold = 0.1f; // NRD_CURVATURE_Z_THRESHOLD
constexpr float kFp16MaxRx = 65504.0f;

// Poisson.hlsli:40-50: offsets of the eight taps and GetGaussianWeight(length) = exp(-0.66 length^2)
#define NRD_B200_POISSON8_X(i) ((i) == 0 ? -0.4706069f : (i) == 1 ? -0.9057375f : (i) == 2 ? -0.3487388f : (i) == 3 ? 0.1023042f : (i) == 4 ? 0.5699277f : (i) == 5 ? 0.2939128f : (i) == 6 ? 0.7836658f : 0.1564120f)
#define NRD_B200_POISSON8_Y(i) ((i) == 0 ? -0.4427112f : (i) == 1 ? 0.3003471f : (i) == 2 ? 0.4037880f : (i) == 3 ? 0.6439373f : (i) == 4 ? 0.3513750f : (i) == 5 ? -0.1131226f : (i) == 6 ? -0.4208784f : -0.8198990f)
#define NRD_B200_POISSON8_GAUSS(i) ((i) == 0 ? 0.7591725f : (i) == 1 ? 0.5482766f : (i) == 2 ? 0.82871586f : (i) == 3 ? 0.75534534f : (i) == 4 ? 0.743887f : (i) == 5 ? 0.9366368f : (i) == 6 ? 0.5931912f : 0.6313964f)

typedef RelaxConstants RC;

__device__ __forceinline__ float Luma(f3 c) { return 0.2126f * c.x + 0.7152f * c.y + 0.0722f * c.z; }
__device__ __forceinline__ float PinnedLuma(f3 c) { return __fadd_rn(__fadd_rn(__fmul_rn(c.x, 0.2126f), __fmul_rn(c.y, 0.7152f)), __fmul_rn(c.z, 0.0722f)); }
__device__ __forceinline__ f3 abs3(f3 a) { return mk3(fabsf(a.x), fabsf(a.y), fabsf(a.z)); }
__device__ __forceinline__ f3 max3(f3 a, f3 b) { return mk3(fmaxf(a.x, b.x), fmaxf(a.y, b.y), fmaxf(a.z, b.z)); }
__device__ __forceinline__ f3 min3(f3 a, f3 b) { return mk3(fminf(a.x, b.x), fminf(a.y, b.y), fminf(a.z, b.z)); }
__device__ __forceinline__ f4 max4(f4 a, float b) { return mk4(fmaxf(a.x, b), fmaxf(a.y, b), fmaxf(a.z, b), fmaxf(a.w, b)); }
__device__ __forceinline__ f4 min4(f4 a, float b) { return mk4(fminf(a.x, b), fminf(a.y, b), fminf(a.z, b), fminf(a.w, b)); }
__device__ __forceinline__ f3 ld3(const float* p) { return mk3(p[0], p[1], p[2]); }
__device__ __forceinline__ float UnpackViewZ(const RC& c, float z) { return fabsf(z * c.gViewZScale); }
__device__ __forceinline__ bool SameMaterial(float m0, float m, float minm) { return fmaxf(m0, minm) == fmaxf(m, minm); }
// exact UNORM8 decode times 255 (history length, material id): decisions depend on it, so keep IEEE division
__device__ __forceinline__ float LoadR8Times255(const Surf& s, int x, int y) { return __fmul_rn(__fdiv_rn((float)LoadU8(s, x, y), 255.0f), 255.0f); }
__device__ __forceinline__ float LoadR8UnormExactClamped(const Surf& s, int x, int y) { return __fdiv_rn((float)LoadU8(s, clampi(x, 0, s.w - 1), clampi(y, 0, s.h - 1)), 255.0f); }
// current-frame guides: the normal comes decoded from the guide surface RELAX_ClassifyTiles filled (one 16-byte load instead of the
// octahedral decode at every tap of every A-trous iteration), roughness / material from the packed bits
#define RX_GUIDE(a, x, y) rb::LoadGuide((a).guide, (a).nr, x, y)
__device__ __forceinline__ bool IsSkyTile(const Surf& tiles, int x, int y) { return LoadU8(tiles, x >> 4, y >> 4) != 0; }
// signal load of a kernel compiled for one or both signals: the absent signal reads as zero and its arithmetic is dead code
template <bool PRESENT> __device__ __forceinline__ f4 LoadSignal(const Surf& s, int x, int y) { return PRESENT ? LoadRGBA16F(s, x, y) : mk4(0.0f); }


// RELAX_Common.hlsli:66-96
__device__ __forceinline__ f3 WorldPosFromClip(const float* R, const float* U, const float* F, float ortho, float csx, float csy, float viewZ)
{
    f3 d = mk3(R[0] * csx - U[0] * csy, R[1] * csx - U[1] * csy, R[2] * csx - U[2] * csy);
    f3 f = ld3(F);
    return ortho == 0.0f ? (f + d) * viewZ : f * viewZ + d;
}
__device__ __forceinline__ f3 CurWorldPosFromClip(const RC& c, float csx, float csy, float z)
{
    return WorldPosFromClip(c.gFrustumRight, c.gFrustumUp, c.gFrustumForward, c.gOrthoMode, csx, csy, z);
}
__device__ __forceinline__ f3 CurWorldPos(const RC& c, int x, int y, float z)
{
    float csx = ((float)x + 0.5f) * c.gRectSizeInv[0] * 2.0f - 1.0f, csy = ((float)y + 0.5f) * c.gRectSizeInv[1] * 2.0f - 1.0f;
    return CurWorldPosFromClip(c, csx, csy, z);
}
// pinned variants for the temporal pass: V.Vprev is evaluated as 1 - cos of a tiny angle there, the result is rounding noise
// unless the whole chain is evaluated with the oracle's operation order
__device__ __forceinline__ f3 PinnedWorldPosFromClip(const float* R, const float* U, const float* F, float ortho, float csx, float csy, float viewZ)
{
    f3 d = mk3(__fadd_rn(__fmul_rn(R[0], csx), -__fmul_rn(U[0], csy)), __fadd_rn(__fmul_rn(R[1], csx), -__fmul_rn(U[1], csy)), __fadd_rn(__fmul_rn(R[2], csx), -__fmul_rn(U[2], csy)));
    if (ortho == 0.0f) return mk3(__fmul_rn(viewZ, __fadd_rn(F[0], d.x)), __fmul_rn(viewZ, __fadd_rn(F[1], d.y)), __fmul_rn(viewZ, __fadd_rn(F[2], d.z)));
    return mk3(__fadd_rn(__fmul_rn(viewZ, F[0]), d.x), __fadd_rn(__fmul_rn(viewZ, F[1]), d.y), __fadd_rn(__fmul_rn(viewZ, F[2]), d.z));
}
__device__ __forceinline__ float PinnedClip(float p, float inv) { return __fadd_rn(__fmul_rn(__fmul_rn(__fadd_rn(p, 0.5f), inv), 2.0f), -1.0f); }
__device__ __forceinline__ f3 PinnedNormalize(f3 v)
{
    float r = __fdiv_rn(1.0f, __fsqrt_rn(PinnedDot3(v.x, v.y, v.z, v)));
    return mk3(__fmul_rn(v.x, r), __fmul_rn(v.y, r), __fmul_rn(v.z, r));
}
// guide decode in the oracle's operation order (NRD.hlsli:600-628): used where a weight is a hard threshold on geometry
__device__ __forceinline__ Guide DecodeGuidePinned(unsigned packed)
{
    float nx = __fadd_rn(__fmul_rn(__fdiv_rn((float)(packed & 1023u), 1023.0f), 2.0f), -1.0f);
    float ny = __fadd_rn(__fmul_rn(__fdiv_rn((float)((packed >> 10) & 1023u), 1023.0f), 2.0f), -1.0f);
    float nz = __fadd_rn(__fadd_rn(1.0f, -fabsf(nx)), -fabsf(ny));
    float t = saturate(-nz);
    nx = __fadd_rn(nx, -__fmul_rn(t, nx >= 0.0f ? 1.0f : -1.0f));
    ny = __fadd_rn(ny, -__fmul_rn(t, ny >= 0.0f ? 1.0f : -1.0f));
    float inv = __fdiv_rn(1.0f, __fsqrt_rn(__fadd_rn(PinnedDot3(nx, ny, nz, mk3(nx, ny, nz)), 1e-9f)));
    Guide g;
    g.N = mk3(__fmul_rn(nx, inv), __fmul_rn(ny, inv), __fmul_rn(nz, inv));
    g.roughness = __fdiv_rn((float)((packed >> 20) & 1023u), 1023.0f);
    g.materialID = __fmul_rn(__fdiv_rn((float)(packed >> 30), 3.0f), 3.0f);
    return g;
}
__device__ __forceinline__ f3 PinnedCurWorldPos(const RelaxConstants& c, int x, int y, float z)
{
    return PinnedWorldPosFromClip(c.gFrustumRight, c.gFrustumUp, c.gFrustumForward, c.gOrthoMode, PinnedClip((float)x, c.gRectSizeInv[0]), PinnedClip((float)y, c.gRectSizeInv[1]), z);
}
__device__ __forceinline__ f3 PinnedAdd(f3 a, f3 b) { return mk3(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y), __fadd_rn(a.z, b.z)); }
__device__ __forceinline__ f3 PinnedSub(f3 a, f3 b) { return mk3(__fadd_rn(a.x, -b.x), __fadd_rn(a.y, -b.y), __fadd_rn(a.z, -b.z)); }
__device__ __forceinline__ f3 PrevWorldPosFromClip(const RC& c, float csx, float csy, float z)
{
    return WorldPosFromClip(c.gPrevFrustumRight, c.gPrevFrustumUp, c.gPrevFrustumForward, c.gOrthoMode, csx, csy, z);
}
__device__ __forceinline__ f3 PrevWorldPos(const RC& c, int x, int y, float z)
{
    float csx = ((float)x + 0.5f) * (1.0f / c.gRectSizePrev[0]) * 2.0f - 1.0f, csy = ((float)y + 0.5f) * (1.0f / c.gRectSizePrev[1]) * 2.0f - 1.0f;
    return PrevWorldPosFromClip(c, csx, csy, z);
}
__device__ __forceinline__ float PixelRadiusToWorld(const RC& c, float pixelRadius, float viewZ) { return pixelRadius * c.gUnproject * lerpf(viewZ, 1.0f, fabsf(c.gOrthoMode)); }
__device__ __forceinline__ float RelaxLobeTanHalfAngle(float roughness, float p = 0.75f) // RELAX_Common.hlsli:112-121
{
    roughness = saturate(roughness);
    p = saturate(p);
    return roughness * roughness * p / (1.0f - p + kEps);
}
__device__ __forceinline__ f2 NormalWeightParamsAtrous(float roughness, float frames, float specConf, float relaxationK, float lobeFraction, float slack) // :123-145
{
    float relaxation = saturate(frames / 5.0f);
    relaxation *= lerpf(1.0f, specConf, relaxationK);
    float f = 0.9f + 0.1f * relaxation;
    float angle = atanf(RelaxLobeTanHalfAngle(roughness, lobeFraction));
    angle *= 10.0f - 9.0f * relaxation;
    angle += slack;
    angle = fminf(1.57079632679f, angle);
    return mk2(angle, f);
}
// :147-156 with the sample's view vector given un-normalised (v = -s / |s|): dot(v0, v) = -dot(v0, s) * rsqrt(dot(s, s))
__device__ __forceinline__ float SpecularNormalWeightAtrousRaw(f2 p0, f3 n0, f3 n, f3 v0, f3 s)
{
    float cosa = fminf(dot(n0, n), -dot(v0, s) * rsqrtf(dot(s, s)));
    float a = AcosApprox(cosa);
    a = SmoothStep(0.0f, p0.x, a);
    return saturate(1.0f - a * p0.y);
}
__device__ __forceinline__ float NormalWeightParam2(float roughness, float angleFraction) // :158-165
{
    return 1.0f / fmaxf(atanf(RelaxLobeTanHalfAngle(roughness, angleFraction)), kNormalUlp);
}
__device__ __forceinline__ float BilateralWeight(float z, float zc) { return LinearStep(0.03f, 0.0f, fabsf(z - zc) / fmaxf(z, zc)); }
__device__ __forceinline__ float PlaneDistWeightAtrous(f3 cw, f3 cn, f3 sw, float thr) { return fabsf(dot(sw - cw, cn)) < thr ? 1.0f : 0.0f; }
__device__ __forceinline__ f3 SafeNormalize(f3 v) { return v * rsqrtf(dot(v, v) + 1e-9f); }
__device__ __forceinline__ f4 UnpackPrevNormalRoughness(f4 p) { return mk4(SafeNormalize(mk3(p.x * 2.0f - 1.0f, p.y * 2.0f - 1.0f, p.z * 2.0f - 1.0f)), p.w); }

__device__ __forceinline__ f4 FetchRGBA8Clamped(const Surf& s, int x, int y) { return UnpackRGBA8(LoadU32(s, clampi(x, 0, s.w - 1), clampi(y, 0, s.h - 1))); }
__device__ __forceinline__ f4 SampleLinearRGBA8(const Surf& s, float u, float v)
{
    float px = u * (float)s.w - 0.5f, py = v * (float)s.h - 0.5f;
    float fx = floorf(px), fy = floorf(py);
    float wx = px - fx, wy = py - fy;
    int x0 = (int)fx, y0 = (int)fy;
    f4 a = lerp4(FetchRGBA8Clamped(s, x0, y0), FetchRGBA8Clamped(s, x0 + 1, y0), wx);
    f4 b = lerp4(FetchRGBA8Clamped(s, x0, y0 + 1), FetchRGBA8Clamped(s, x0 + 1, y0 + 1), wx);
    return lerp4(a, b, wy);
}
__device__ __forceinline__ f2 ScreenUvNoKill(const float* m, f3 X)
{
    float cx = PinnedRow(m, 0, X.x, X.y, X.z), cy = PinnedRow(m, 1, X.x, X.y, X.z), cw = PinnedRow(m, 3, X.x, X.y, X.z);
    return mk2(__fadd_rn(__fmul_rn(__fdiv_rn(cx, cw), 0.5f), 0.5f), __fadd_rn(__fmul_rn(__fdiv_rn(cy, cw), -0.5f), 0.5f));
}
__device__ __forceinline__ float ParallaxInPixels(f3 X, f2 uv0, const float* m, float w, float h)
{
    f2 uv = GetScreenUv(m, X);
    float dx = (uv.x - uv0.x) * w, dy = (uv.y - uv0.y) * h;
    return sqrtf(dx * dx + dy * dy);
}
__device__ __forceinline__ float ThinLens(float O, float curvature) { return O / (2.0f * curvature * O + 1.0f); }
// thin-lens virtual position (Common.hlsli:404-461)
__device__ __forceinline__ f3 XvirtualRx(float hitDist, float curvature, f3 X, f3 Xprev, f3 N, f3 V, float roughness)
{
    f4 D = SpecularDominantDirection(N, V, roughness);
    f3 ray = xyz(D) * hitDist;
    f3 T, B;
    GetBasis(N, T, B);
    float Oz = -dot(N, ray);
    float Ox = dot(T, ray), Oy = dot(B, ray);
    float mag = 1.0f / (2.0f * curvature * Oz - 1.0f);
    float f = length(X) * (1.0f - fabsf(dot(N, V))) * fmaxf(curvature, 0.0f);
    mag *= 1.0f / (1.0f + f);
    float lenI = sqrtf(Ox * Ox + Oy * Oy + Oz * Oz) * fabsf(mag);
    f3 Iw = V * lenI;
    float closeness = saturate(length(Iw) / (hitDist + kEps));
    f3 origin = lerp3(Xprev, X, closeness * D.w);
    return origin - Iw * D.w;
}
__device__ __forceinline__ f3 RgbToYCoCg(f3 c) { return mk3(0.25f * c.x + 0.5f * c.y + 0.25f * c.z, 0.5f * c.x - 0.5f * c.z, -0.25f * c.x + 0.5f * c.y - 0.25f * c.z); }
__device__ __forceinline__ f3 YCoCgToRgb(f3 c)
{
    float t = c.x - c.z;
    return max3(mk3(t + c.y, c.x + c.z, t - c.y), mk3(0.0f));
}

// =============================================================================================
// Classify tiles (RELAX_ClassifyTiles.cs.hlsl:18-49): one warp per 16x16 tile
// =============================================================================================
struct RxTilesArgs
{
    Surf z, tiles, nr, guide;
    float denoisingRange;
    int tilesW, tilesH;
    int buildGuide; // also decode IN_NORMAL_ROUGHNESS of the tile into the guide surface (surf.h PassLaunch::guide)
};
__global__ void __launch_bounds__(256) RelaxClassifyTilesKernel(const __grid_constant__ RxTilesArgs a)
{
    int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (warp >= a.tilesW * a.tilesH) return;
    int tx = warp % a.tilesW, ty = warp / a.tilesW;
    const bool ownTile = ty >= a.tiles.y0 && ty < a.tiles.y1;
    // tiles of another strip: only their rows that this rank holds as ghost rows matter (guide build, see below)
    if (!ownTile && (!a.buildGuide || ty * 16 + 15 < a.guide.ly0 || ty * 16 >= a.guide.ly0 + (int)a.guide.lrows)) return;
    bool allSky = true;
#pragma unroll
    for (int k = 0; k < 8; k++)
    {
        int i = k * 32 + lane;
        int x = tx * 16 + (i & 15), y = ty * 16 + (i >> 4);
        float z = 0.0f;
        if (Inside(a.z, x, y))
        {
            // the guide is built for every row held locally: the ghost rows of IN_VIEWZ / IN_NORMAL_ROUGHNESS arrived with the
            // frame-start push, so the guide's ghost rows are decoded here instead of being sent by the neighbour
            const bool held = a.buildGuide && (unsigned)(y - a.guide.ly0) < a.guide.lrows;
            if (ownTile || held) z = LoadR32F(Near(a.z), x, y);
            if (held) StoreRGBA32F(a.guide, x, y, mk4(rb::DecodeNormalExact(LoadU32(Near(a.nr), x, y)), z));
        }
        allSky = allSky && (fabsf(z) > a.denoisingRange);
    }
    allSky = __all_sync(0xffffffffu, allSky);
    if (lane == 0 && ownTile) StoreU8(a.tiles, tx, ty, allSky ? 255u : 0u);
}

// =============================================================================================
// Hit-distance reconstruction (RELAX_HitDistReconstruction.hlsli:10-155): RelaxSettings::hitDistanceReconstructionMode 3x3 / 5x5.
// A dense (2 BORDER + 1)^2 stencil over guides and hit distances; the neighbourhood of a 32x8 CTA is read through L1 (every texel
// is shared by up to 25 threads of the CTA).
// =============================================================================================
struct RxHitDistArgs
{
    RC c;
    Surf tiles, spec, diff, nr, z, outSpec, outDiff;
    Surf guide;
    int rowBegin, rowEnd;
};
template <bool DIFF, bool SPEC, int BORDER> __global__ void __launch_bounds__(256) RelaxHitDistReconstructionKernel(const __grid_constant__ RxHitDistArgs a)
{
    const RC& c = a.c;
    const int x = blockIdx.x * 32 + threadIdx.x, y = a.rowBegin + blockIdx.y * 8 + threadIdx.y;
    const int W = c.gRectSize[0], H = c.gRectSize[1];
    if (x >= W || y >= H || y >= a.rowEnd) return;
    if (IsSkyTile(a.tiles, x, y)) return;
    const float centerViewZ = UnpackViewZ(c, LoadR32F(a.z, x, y));
    if (centerViewZ > c.gDenoisingRange) return;
    const Guide g = RX_GUIDE(a, x, y);
    const f4 centerSpec = LoadSignal<SPEC>(a.spec, x, y), centerDiff = LoadSignal<DIFF>(a.diff, x, y);
    // GetNormalWeightParam(1, 1, roughness) (Common.hlsli:486-500): 1 / max(atan(lobe tan half angle at 75 % of the volume), encoding error)
    const float specularNormalWeightParam = 1.0f / fmaxf(atanf(LobeTanHalfAngle(g.roughness, kLobeVolume)), kNormalEncodingError);
    const float diffuseNormalWeightParam = 1.0f / fmaxf(atanf(LobeTanHalfAngle(1.0f, kLobeVolume)), kNormalEncodingError);
    // (sic) the reference weighs every tap by the roughness of the CENTRE against itself (:117): one factor for all taps
    const f2 rrp = RelaxedRoughnessWeightParams(g.roughness * g.roughness, 1.0f);
    const float roughnessWeight = ExpWeight(g.roughness * g.roughness, rrp.x, rrp.y);
    float sumSpecularWeight = centerSpec.w != 0.0f ? 1000.0f : 0.0f, sumDiffuseWeight = centerDiff.w != 0.0f ? 1000.0f : 0.0f;
    float sumSpecularHitDist = centerSpec.w * sumSpecularWeight, sumDiffuseHitDist = centerDiff.w * sumDiffuseWeight;
#pragma unroll
    for (int dy = -BORDER; dy <= BORDER; dy++)
#pragma unroll
        for (int dx = -BORDER; dx <= BORDER; dx++)
        {
            if (dx == 0 && dy == 0) continue;
            const int px = x + dx, py = y + dy;
            if ((unsigned)px >= (unsigned)W || (unsigned)py >= (unsigned)H) continue; // IsInScreenNearest of the neighbour's centre
            const float4 q = __ldg(TexelPtr<float4>(a.guide, px, py)); // {N.xyz, raw viewZ}
            const float sampleViewZ = fabsf(q.w * c.gViewZScale);
            float w = sampleViewZ < c.gDenoisingRange ? __expf(-0.66f * 0.25f * (float)(dx * dx + dy * dy)) : 0.0f; // GetGaussianWeight(length(o) / 2)
            w *= BilateralWeight(sampleViewZ, centerViewZ);
            const float angle = AcosApprox(g.N.x * q.x + g.N.y * q.y + g.N.z * q.z);
            if (SPEC)
            {
                float ws = w * ExpWeight(angle, specularNormalWeightParam, 0.0f) * roughnessWeight;
                const float h = ws == 0.0f ? 0.0f : LoadSignal<SPEC>(a.spec, px, py).w;
                ws = h != 0.0f ? ws : 0.0f;
                sumSpecularHitDist = fmaf(h, ws, sumSpecularHitDist);
                sumSpecularWeight += ws;
            }
            if (DIFF)
            {
                float wd = w * ExpWeight(angle, diffuseNormalWeightParam, 0.0f);
                const float h = wd == 0.0f ? 0.0f : LoadSignal<DIFF>(a.diff, px, py).w;
                wd = h != 0.0f ? wd : 0.0f;
                sumDiffuseHitDist = fmaf(h, wd, sumDiffuseHitDist);
                sumDiffuseWeight += wd;
            }
        }
    if (SPEC) StoreRGBA16F(a.outSpec, x, y, mk4(xyz(centerSpec), sumSpecularHitDist / fmaxf(sumSpecularWeight, 1e-6f)));
    if (DIFF) StoreRGBA16F(a.outDiff, x, y, mk4(xyz(centerDiff), sumDiffuseHitDist / fmaxf(sumDiffuseWeight, 1e-6f)));
}

// =============================================================================================
// Pre-pass (RELAX_PrePass.hlsli:13-347).  CB = a checkerboarded input (RelaxSettings::checkerboardMode): the signal is packed into the
// left half of its texture, pixels without data are resolved from their left / right neighbours before the blur (:28-58, :73-110),
// taps that land on a pixel without data move one pixel sideways (ApplyCheckerboardShift)
// =============================================================================================
struct RxPrePassArgs
{
    RC c;
    Surf tiles, spec, diff, nr, z, outSpec, outDiff;
    Surf guide; // decoded guides of the current frame (surf.h PassLaunch::guide)
    int rowBegin, rowEnd;
};
template <bool DIFF, bool SPEC, bool CB = false> __global__ void __launch_bounds__(256) RelaxPrePassKernel(const __grid_constant__ RxPrePassArgs a)
{
    const RC& c = a.c;
    const int x = blockIdx.x * 32 + threadIdx.x, y = a.rowBegin + blockIdx.y * 8 + threadIdx.y;
    const int W = c.gRectSize[0], H = c.gRectSize[1];
    if (x >= W || y >= H || y >= a.rowEnd) return;
    if (IsSkyTile(a.tiles, x, y)) return;
    const float centerViewZ = UnpackViewZ(c, LoadR32F(a.z, x, y));
    if (centerViewZ > c.gDenoisingRange) return;

    const Guide g = RX_GUIDE(a, x, y);
    const f3 centerNormal = g.N;
    const float centerRoughness = g.roughness;
    const f3 centerWorldPos = CurWorldPos(c, x, y, centerViewZ);
    const float rx0 = c.gRotatorPre[0], rx1 = c.gRotatorPre[1], rx2 = c.gRotatorPre[2], rx3 = c.gRotatorPre[3];
    const f2 pixelUv = PixelUv(x, y, c.gRectSizeInv);
    const float posX = __fmul_rn(pixelUv.x, (float)W), posY = __fmul_rn(pixelUv.y, (float)H);
    const float planeZ = c.gOrthoMode == 0.0f ? centerViewZ : 1.0f;
    const float frustumSize = PixelRadiusToWorld(c, (float)min(W, H), centerViewZ);

    // checkerboard resolve weights (:28-58)
    unsigned checkerboard = 0u;
    int cbX0 = 0, cbX1 = 0;
    float cbW0 = 1.0f, cbW1 = 1.0f, cbMat0 = 0.0f, cbMat1 = 0.0f;
    if (CB)
    {
        checkerboard = CheckerBoard(x, y, c.gFrameIndex);
        const int x0 = max(x - 1, 0), x1 = min(x + 1, W - 1);
        const float viewZ0 = UnpackViewZ(c, LoadR32F(a.z, x0, y)), viewZ1 = UnpackViewZ(c, LoadR32F(a.z, x1, y));
        cbMat0 = (float)(LoadU32(a.nr, x0, y) >> 30);
        cbMat1 = (float)(LoadU32(a.nr, x1, y) >> 30);
        cbW0 = (viewZ0 > c.gDenoisingRange || x < 1) ? 0.0f : BilateralWeight(viewZ0, centerViewZ);
        cbW1 = (viewZ1 > c.gDenoisingRange || x > W - 2) ? 0.0f : BilateralWeight(viewZ1, centerViewZ);
        cbX0 = x0 >> 1;
        cbX1 = x1 >> 1;
    }
    auto resolve = [&](const Surf& signal, float minMaterial) {
        float w0 = SameMaterial(g.materialID, cbMat0, minMaterial) ? cbW0 : 0.0f, w1 = SameMaterial(g.materialID, cbMat1, minMaterial) ? cbW1 : 0.0f;
        const float norm = PositiveRcp(w0 + w1);
        w0 *= norm;
        w1 *= norm;
        f4 s0 = LoadRGBA16F(signal, cbX0, y), s1 = LoadRGBA16F(signal, cbX1, y);
        s0 = w0 == 0.0f ? mk4(0.0f) : s0;
        s1 = w1 == 0.0f ? mk4(0.0f) : s1;
        return s0 * w0 + s1 * w1;
    };

    // tap position in pixels (pinned: selects the texel), returns the in-screen flag
    // (the rotated offsets are per-frame uniforms: with the tap index a compile-time constant of the unrolled loops they fold into
    // uniform-datapath arithmetic; floor() is the FADD.RM trick of the REBLUR filters -- same value for |x| < 2^22, off screen otherwise)
    const float kx2 = 2.0f * c.gRectSizeInv[0], ky2 = 2.0f * c.gRectSizeInv[1];
    auto tapPos = [&](int i, float blurRadius, unsigned mode, int& tx, int& ty, float& csx, float& csy) {
        const float ox = NRD_B200_POISSON8_X(i), oy = NRD_B200_POISSON8_Y(i);
        const float rxv = __fadd_rn(__fmul_rn(ox, rx0), __fmul_rn(oy, rx1)), ryv = __fadd_rn(__fmul_rn(ox, rx2), __fmul_rn(oy, rx3));
        int ix, iy;
        float fx = FloorIndex(__fadd_rn(posX, __fmul_rn(rxv, blurRadius)), ix);
        const float fy = FloorIndex(__fadd_rn(posY, __fmul_rn(ryv, blurRadius)), iy);
        if (CB && mode != 2u && CheckerBoard(ix, iy, c.gFrameIndex) != mode)
        {
            const int d = (i & 1) == 0 ? -1 : 1; // ApplyCheckerboardShift: even taps move left, odd taps right
            ix += d;
            fx += (float)d;
        }
        const bool inScreen = (unsigned)ix < (unsigned)W && (unsigned)iy < (unsigned)H;
        tx = clampi(ix, 0, W - 1);
        ty = clampi(iy, 0, H - 1);
        csx = fmaf(fx + 0.5f, kx2, -1.0f);
        csy = fmaf(fy + 0.5f, ky2, -1.0f);
        return inScreen;
    };

    // ---- diffuse
    if (DIFF)
    {
        const int half = CB && c.gDiffCheckerboard != 2u ? 1 : 0;
        f4 diff = LoadRGBA16F(a.diff, x >> half, y);
        if (CB && half && checkerboard != c.gDiffCheckerboard) diff = resolve(a.diff, c.gDiffMinMaterial);
        if (c.gDiffBlurRadius > 0.0f)
        {
            float hitDist = diff.w == 0.0f ? 1.0f : diff.w;
            float blurRadius = c.gDiffBlurRadius * saturate(hitDist / frustumSize);
            if (diff.w == 0.0f) blurRadius = fmaxf(blurRadius, 1.0f);
            const float normalWeightParam = NormalWeightParam2(1.0f, 0.25f * c.gLobeAngleFraction);
            const f2 hdp = HitDistanceWeightParams(diff.w, 1.0f / 9.0f, SpecMagicCurve(1.0f));
            float weightSum = 1.0f;
            const float planeThreshold = c.gDepthThreshold * planeZ, planeC = dot(centerWorldPos, centerNormal);
#pragma unroll
            for (int i = 0; i < 8; i++)
            {
                int tx, ty;
                float csx, csy;
                const bool inScreen = tapPos(i, blurRadius, c.gDiffCheckerboard, tx, ty, csx, csy);
                const float4 q = __ldg(TexelPtr<float4>(a.guide, tx, ty)); // {N.xyz, raw viewZ}
                const float sz = fabsf(q.w * c.gViewZScale);
                const f3 sw = CurWorldPosFromClip(c, csx, csy, sz);
                float w = inScreen && sz < c.gDenoisingRange ? NRD_B200_POISSON8_GAUSS(i) : 0.0f;
                if (c.gDiffMinMaterial < 3.0f) w = SameMaterial(g.materialID, (float)(LoadU32(a.nr, tx, ty) >> 30), c.gDiffMinMaterial) ? w : 0.0f;
                w = fabsf(dot(sw, centerNormal) - planeC) > planeThreshold ? 0.0f : w;
                w *= NonExpWeight(AcosApprox(centerNormal.x * q.x + centerNormal.y * q.y + centerNormal.z * q.z), normalWeightParam, 0.0f);
                if (w != 0.0f)
                {
                    const f4 s = LoadRGBA16F(a.diff, tx >> half, ty);
                    w *= lerpf(c.gMinHitDistanceWeight, 1.0f, ExpWeight(s.w, hdp.x, hdp.y));
                    weightSum += w;
                    diff = diff + s * w;
                }
            }
            diff = mk4(diff.x / weightSum, diff.y / weightSum, diff.z / weightSum, diff.w / weightSum);
        }
        StoreRGBA16F(a.outDiff, x, y, min4(max4(diff, 0.0f), kFp16MaxRx));
    }
    // ---- specular
    if (SPEC)
    {
        const int half = CB && c.gSpecCheckerboard != 2u ? 1 : 0;
        f4 spec = LoadRGBA16F(a.spec, x >> half, y);
        if (CB && half && checkerboard != c.gSpecCheckerboard) spec = resolve(a.spec, c.gSpecMinMaterial);
        spec.w = fmaxf(0.0f, fminf(c.gDenoisingRange, spec.w));
        if (c.gSpecBlurRadius > 0.0f)
        {
            f3 V = c.gOrthoMode == 0.0f ? normalize(-centerWorldPos) : ld3(c.gFrustumForward);
            f4 D = SpecularDominantDirection(centerNormal, V, centerRoughness);
            float NoD = fabsf(dot(centerNormal, xyz(D)));
            float hitDist = spec.w == 0.0f ? 1.0f : spec.w;
            float hitDistFactor = saturate(hitDist * NoD / frustumSize);
            float smc = SpecMagicCurve(centerRoughness);
            float blurRadius = c.gSpecBlurRadius * hitDistFactor * smc;
            float lobeRadius = hitDist * NoD * LobeTanHalfAngle(centerRoughness, 0.75f);
            float minBlurRadius = lobeRadius / PixelRadiusToWorld(c, 1.0f, centerViewZ + hitDist * D.w);
            blurRadius = fminf(blurRadius, minBlurRadius);
            if (spec.w == 0.0f) blurRadius = fmaxf(blurRadius, 1.0f);
            const float normalWeightParam = NormalWeightParam2(centerRoughness, 0.5f * c.gLobeAngleFraction);
            const f2 hdp = HitDistanceWeightParams(spec.w, 1.0f / 9.0f, smc);
            const f2 rwp = RoughnessWeightParams(centerRoughness, c.gRoughnessFraction);
            const float minHitDistWeight = spec.w == 0.0f ? 1.0f : c.gMinHitDistanceWeight * smc;
            float specularHitT = spec.w == 0.0f ? c.gDenoisingRange : spec.w;
            float minHitT = specularHitT == 0.0f ? kInf : specularHitT;
            const float roughnessLerp = LinearStep(0.5f, 1.0f, centerRoughness);
            float weightSum = 1.0f;
            const float planeThreshold = c.gDepthThreshold * planeZ, planeC = dot(centerWorldPos, centerNormal);
            const float rwpx = rwp.x * (1.0f / 1023.0f); // applied to the tap's 10-bit roughness code
#pragma unroll
            for (int i = 0; i < 8; i++)
            {
                int tx, ty;
                float csx, csy;
                const bool inScreen = tapPos(i, blurRadius, c.gSpecCheckerboard, tx, ty, csx, csy);
                const float4 q = __ldg(TexelPtr<float4>(a.guide, tx, ty)); // {N.xyz, raw viewZ}
                const unsigned packed = LoadU32(a.nr, tx, ty);
                const float sz = fabsf(q.w * c.gViewZScale);
                float w = inScreen && sz < c.gDenoisingRange ? NRD_B200_POISSON8_GAUSS(i) : 0.0f;
                if (c.gSpecMinMaterial < 3.0f) w = SameMaterial(g.materialID, (float)(packed >> 30), c.gSpecMinMaterial) ? w : 0.0f;
                w *= NonExpWeight((float)((packed >> 20) & 1023u), rwpx, rwp.y);
                w *= NonExpWeight(AcosApprox(centerNormal.x * q.x + centerNormal.y * q.y + centerNormal.z * q.z), normalWeightParam, 0.0f);
                const f3 sw = CurWorldPosFromClip(c, csx, csy, sz);
                w = fabsf(dot(sw, centerNormal) - planeC) > planeThreshold ? 0.0f : w;
                if (w != 0.0f)
                {
                    const f4 s = LoadRGBA16F(a.spec, tx >> half, ty);
                    w *= lerpf(minHitDistWeight, 1.0f, ExpWeight(s.w, hdp.x, hdp.y));
                    const float d = length(sw - centerWorldPos);
                    w *= lerpf(SatMul(s.w, __fdividef(1.0f, spec.w + d)), 1.0f, roughnessLerp);
                    weightSum += w;
                    spec.x += s.x * w;
                    spec.y += s.y * w;
                    spec.z += s.z * w;
                    if (w != 0.0f) minHitT = fminf(minHitT, s.w == 0.0f ? kInf : s.w);
                }
            }
            spec.x /= weightSum;
            spec.y /= weightSum;
            spec.z /= weightSum;
            spec.w = minHitT == kInf ? 0.0f : minHitT;
        }
        StoreRGBA16F(a.outSpec, x, y, min4(max4(spec, 0.0f), kFp16MaxRx));
    }
}

// =============================================================================================
// Temporal accumulation (RELAX_TemporalAccumulation.hlsli:11-930)
// =============================================================================================
struct RxTaArgs
{
    RC c;
    Surf tiles, spec, diff, mv, nr, z, histSpecFast, histDiffFast, histSpec, histDiff, prevNr, prevZ, prevHitDist, prevLength, prevMaterial;
    Surf specConfidence, diffConfidence, mix; // optional R8_UNORM inputs, read only when the constants say so
    Surf outSpec, outDiff, outSpecFast, outDiffFast, outHitDist, outLength, outConfidence;
    Surf guide; // decoded guides of the current frame (surf.h PassLaunch::guide)
    int rowBegin, rowEnd;
};
template <bool DIFF, bool SPEC, bool CB = false> __global__ void __launch_bounds__(128, 5) RelaxTemporalAccumulationKernel(const __grid_constant__ RxTaArgs a)
{
    const RC& c = a.c;
    const int x = blockIdx.x * 32 + threadIdx.x, y = a.rowBegin + blockIdx.y * 4 + threadIdx.y;
    const int W = c.gRectSize[0], H = c.gRectSize[1];
    if (x >= W || y >= H || y >= a.rowEnd) return;
    if (IsSkyTile(a.tiles, x, y)) return;
    const float currentLinearZ = UnpackViewZ(c, LoadR32F(a.z, x, y));
    if (currentLinearZ > c.gDenoisingRange) return;
    const float fW = (float)W, fH = (float)H;

    const Guide g = RX_GUIDE(a, x, y);
    const f3 currentNormal = g.N;
    const float currentRoughness = g.roughness;
    const float currentMaterialID = g.materialID;
    const f3 currentWorldPos = PinnedWorldPosFromClip(c.gFrustumRight, c.gFrustumUp, c.gFrustumForward, c.gOrthoMode, PinnedClip((float)x, c.gRectSizeInv[0]),
                                                      PinnedClip((float)y, c.gRectSizeInv[1]), currentLinearZ);
    const f3 fwd = ld3(c.gFrustumForward);
    const f3 currentViewVector = c.gOrthoMode == 0.0f ? currentWorldPos : normalize(fwd) * currentLinearZ;
    const f3 V = -PinnedNormalize(currentViewVector);
    const float NoV = fabsf(dot(currentNormal, V));
    const f3 cameraDelta = ld3(c.gCameraDelta);

    // ---- motion (pinned: prevUVSMB selects the history footprint)
    const f2 pixelUv = PixelUv(x, y, c.gRectSizeInv);
    f4 mvRaw = LoadRGBA16F(a.mv, x, y);
    f3 mv = mk3(__fmul_rn(mvRaw.x, c.gMvScale[0]), __fmul_rn(mvRaw.y, c.gMvScale[1]), __fmul_rn(mvRaw.z, c.gMvScale[2]));
    f3 prevWorldPos = currentWorldPos;
    f2 prevUVSMB = mk2(__fadd_rn(pixelUv.x, mv.x), __fadd_rn(pixelUv.y, mv.y));
    if (c.gMvScale[3] == 0.0f)
    {
        if (c.gMvScale[2] == 0.0f) mv.z = __fadd_rn(AffineTransform(c.gWorldToViewPrev, currentWorldPos).z, -currentLinearZ);
        prevWorldPos = PinnedAdd(PinnedWorldPosFromClip(c.gPrevFrustumRight, c.gPrevFrustumUp, c.gPrevFrustumForward, c.gOrthoMode, __fadd_rn(__fmul_rn(prevUVSMB.x, 2.0f), -1.0f),
                                                        __fadd_rn(__fmul_rn(prevUVSMB.y, 2.0f), -1.0f), __fadd_rn(currentLinearZ, mv.z)),
                                 cameraDelta);
    }
    else
    {
        prevWorldPos = PinnedAdd(prevWorldPos, mv);
        prevUVSMB = GetScreenUv(c.gWorldToClipPrev, prevWorldPos);
    }

    const f3 diffuseIllumination = DIFF ? xyz(LoadRGBA16F(a.diff, x, y)) : mk3(0.0f);
    const f4 specularIllumination = SPEC ? LoadRGBA16F(a.spec, x, y) : mk4(0.0f);

    // ---- 3x3: min hit distance and average normal (shared-memory preload in the reference, :360-374)
    float minHitDist3x3 = specularIllumination.w == 0.0f ? kInf : specularIllumination.w;
    f3 currentNormalAveraged = currentNormal;
    f3 n10 = currentNormal, n01 = currentNormal;
#pragma unroll
    for (int i = -1; i <= 1; i++)
#pragma unroll
        for (int j = -1; j <= 1; j++)
        {
            if (i == 0 && j == 0) continue;
            int px = clampi(x + i, 0, W - 1), py = clampi(y + j, 0, H - 1);
            f3 n = RX_GUIDE(a, px, py).N;
            const float h = SPEC ? LoadRGBA16F(a.spec, px, py).w : 0.0f;
            minHitDist3x3 = fminf(minHitDist3x3, h == 0.0f ? kInf : h);
            currentNormalAveraged = currentNormalAveraged + n;
            if (i == 1 && j == 0) n10 = n;
            if (i == 0 && j == 1) n01 = n;
        }
    currentNormalAveraged = currentNormalAveraged * (1.0f / 9.0f);
    const float currentRoughnessModified = ModifiedRoughness(currentRoughness, currentNormalAveraged);

    const float specular1stMoment = Luma(xyz(specularIllumination));
    const float specular2ndMoment = specular1stMoment * specular1stMoment;
    const float diffuse1stMoment = Luma(diffuseIllumination);
    const float diffuse2ndMoment = diffuse1stMoment * diffuse1stMoment;

    const float smbParallaxInPixels1 = ParallaxInPixels(PinnedAdd(prevWorldPos, cameraDelta), c.gOrthoMode == 0.0f ? prevUVSMB : pixelUv, c.gWorldToClipPrev, fW, fH);
    const float smbParallaxInPixels2 = ParallaxInPixels(PinnedSub(prevWorldPos, cameraDelta), c.gOrthoMode == 0.0f ? pixelUv : prevUVSMB, c.gWorldToClip, fW, fH);
    const float smbParallaxInPixelsMax = fmaxf(smbParallaxInPixels1, smbParallaxInPixels2);
    const float smbParallaxInPixelsMin = fminf(smbParallaxInPixels1, smbParallaxInPixels2);
    const float pixelSize = PixelRadiusToWorld(c, 1.0f, currentLinearZ);

    float disocclusionThresholdMix = 0.0f;
    if (currentMaterialID == c.gStrandMaterialID) disocclusionThresholdMix = pixelSize / (pixelSize + c.gStrandThickness);
    if (c.gHasDisocclusionThresholdMix) disocclusionThresholdMix = LoadR8Unorm(Near(a.mix), x, y);
    const float disocclusionThreshold = lerpf(c.gDisocclusionThreshold, c.gDisocclusionThresholdAlternate, disocclusionThresholdMix);

    // ================= surface motion based history (:35-229)
    float footprintQuality, historyLength, prevReflectionHitTSMB, SMBReprojectionFound;
    f4 prevDiffSMB, prevSpecSMB;
    f3 prevDiffSMBResponsive, prevSpecSMBResponsive;
    {
        const f3 currentNormalN = normalize(currentNormalAveraged);
        const f2 prevPixelPos = mk2(__fmul_rn(prevUVSMB.x, c.gRectSizePrev[0]), __fmul_rn(prevUVSMB.y, c.gRectSizePrev[1]));
        const float tx = __fadd_rn(prevPixelPos.x, -0.5f), ty = __fadd_rn(prevPixelPos.y, -0.5f);
        const float box = floorf(tx), boy = floorf(ty);
        const float bwx = __fadd_rn(tx, -box), bwy = __fadd_rn(ty, -boy);
        const int bx = (int)fmaxf(fminf(box, 1e8f), -1e8f), by = (int)fmaxf(fminf(boy, 1e8f), -1e8f);
        const int zw = a.prevZ.w - 1, zh = a.prevZ.h - 1;

        const float frustumSize = pixelSize * (float)min(W, H);
        const float slopeScale = 1.0f / lerpf(lerpf(0.05f, 1.0f, NoV), 1.0f, saturate(smbParallaxInPixelsMax / 30.0f));
        const float thrBase = saturate(disocclusionThreshold * slopeScale) * frustumSize;
        const float ix0 = (box >= 0.0f && box < c.gRectSizePrev[0]) ? 1.0f : 0.0f, ix1 = (box + 1.0f >= 0.0f && box + 1.0f < c.gRectSizePrev[0]) ? 1.0f : 0.0f;
        const float iy0 = (boy >= 0.0f && boy < c.gRectSizePrev[1]) ? 1.0f : 0.0f, iy1 = (boy + 1.0f >= 0.0f && boy + 1.0f < c.gRectSizePrev[1]) ? 1.0f : 0.0f;
        const float thr[4] = {thrBase * (ix0 * iy0) - kEps, thrBase * (ix1 * iy0) - kEps, thrBase * (ix0 * iy1) - kEps, thrBase * (ix1 * iy1) - kEps};
        const float prevViewZ = AffineTransform(c.gWorldToViewPrev, prevWorldPos).z;
        const float minMaterialID = fminf(c.gSpecMinMaterial, c.gDiffMinMaterial);

        // 4x4 footprint (bx-1 .. bx+2) without the corners; quadrant q = (i>=1) + 2*(j>=1) picks the threshold
        float validSum = 0.0f;
        float v00 = 0.0f, v10 = 0.0f, v01 = 0.0f, v11 = 0.0f;
#pragma unroll
        for (int j = 0; j < 4; j++)
#pragma unroll
            for (int i = 0; i < 4; i++)
            {
                if ((i == 0 || i == 3) && (j == 0 || j == 3)) continue;
                int px = clampi(bx - 1 + i, 0, zw), py = clampi(by - 1 + j, 0, zh);
                float z = UnpackViewZ(c, LoadR32F(a.prevZ, px, py));
                float m = LoadR8Times255(a.prevMaterial, px, py);
                float t = thr[(i >> 1) + 2 * (j >> 1)];
                float v = fabsf(z - prevViewZ) <= t ? 1.0f : 0.0f;
                v *= SameMaterial(currentMaterialID, m, minMaterialID) ? 1.0f : 0.0f;
                validSum += v;
                if (i == 1 && j == 1) v00 = v;
                if (i == 2 && j == 1) v10 = v;
                if (i == 1 && j == 2) v01 = v;
                if (i == 2 && j == 2) v11 = v;
            }
        float bicubicFootprintValid = validSum > 11.5f ? 1.0f : 0.0f;
        f4 tapsValid = mk4(v00, v10, v01, v11);

        const float un = (box + 1.0f) * c.gResourceSizeInvPrev[0], vn = (boy + 1.0f) * c.gResourceSizeInvPrev[1];
        f3 prevNormalFlat = xyz(UnpackPrevNormalRoughness(SampleLinearRGBA8(a.prevNr, un, vn)));
        prevNormalFlat = Rotate(c.gWorldPrevToWorld, prevNormalFlat);
        if (dot(currentNormalN, prevNormalFlat) < 0.0f)
        {
            tapsValid = mk4(0.0f);
            bicubicFootprintValid = 0.0f;
        }
        const float omx = 1.0f - bwx, omy = 1.0f - bwy;
        const f4 bcw = mk4(tapsValid.x * (omx * omy), tapsValid.y * (bwx * omy), tapsValid.z * (omx * bwy), tapsValid.w * (bwx * bwy));
        const bool useBicubic = bicubicFootprintValid > 0.0f;
        const CatRomSetup cr = SetupCatRom(prevPixelPos, c.gResourceSizeInvPrev, bcw, useBicubic);
        prevDiffSMB = DIFF ? max4(ResolveCatRom4<false>(cr, a.histDiff), 0.0f) : mk4(0.0f);
        prevSpecSMB = SPEC ? max4(ResolveCatRom4<false>(cr, a.histSpec), 0.0f) : mk4(0.0f);
        prevDiffSMBResponsive = DIFF ? xyz(max4(ResolveCatRom4<false>(cr, a.histDiffFast), 0.0f)) : mk3(0.0f);
        prevSpecSMBResponsive = SPEC ? xyz(max4(ResolveCatRom4<false>(cr, a.histSpecFast), 0.0f)) : mk3(0.0f);

        const float wsum = bcw.x + bcw.y + bcw.z + bcw.w;
        {
            // the reference filters the [0,1] value and scales by 255 afterwards; keep that order
            float s00 = LoadR8UnormExactClamped(a.prevLength, bx, by), s10 = LoadR8UnormExactClamped(a.prevLength, bx + 1, by);
            float s01 = LoadR8UnormExactClamped(a.prevLength, bx, by + 1), s11 = LoadR8UnormExactClamped(a.prevLength, bx + 1, by + 1);
            float o = s00 * bcw.x + s10 * bcw.y + s01 * bcw.z + s11 * bcw.w;
            historyLength = 255.0f * (wsum < 0.0001f ? 0.0f : o / wsum);
        }
        prevReflectionHitTSMB = 0.0f;
        if (SPEC)
        {
            float s00 = FetchClamped1(a.prevHitDist, bx, by), s10 = FetchClamped1(a.prevHitDist, bx + 1, by);
            float s01 = FetchClamped1(a.prevHitDist, bx, by + 1), s11 = FetchClamped1(a.prevHitDist, bx + 1, by + 1);
            float o = s00 * bcw.x + s10 * bcw.y + s01 * bcw.z + s11 * bcw.w;
            prevReflectionHitTSMB = fmaxf(0.001f, wsum < 0.0001f ? 0.0f : o / wsum);
        }
        SMBReprojectionFound = useBicubic ? 2.0f : 1.0f;
        footprintQuality = useBicubic ? 1.0f : wsum;
        if (!(tapsValid.x != 0.0f || tapsValid.y != 0.0f || tapsValid.z != 0.0f || tapsValid.w != 0.0f))
        {
            SMBReprojectionFound = 0.0f;
            footprintQuality = 0.0f;
        }
    }

    historyLength = fminf(kMaxAccumRelax, historyLength + 1.0f);
    const f3 Vprev = c.gOrthoMode == 0.0f ? -PinnedNormalize(PinnedSub(prevWorldPos, cameraDelta)) : -normalize(ld3(c.gPrevFrustumForward));
    const float NoVprev = fabsf(dot(currentNormal, Vprev));
    float sizeQuality = (NoVprev + 1e-3f) / (NoV + 1e-3f);
    sizeQuality *= sizeQuality;
    sizeQuality *= sizeQuality;
    footprintQuality *= lerpf(0.1f, 1.0f, saturate(sizeQuality + fabsf(c.gOrthoMode)));
    if (footprintQuality < 1.0f)
    {
        historyLength *= sqrtf(footprintQuality);
        historyLength = fmaxf(historyLength, 1.0f);
    }
    historyLength = c.gResetHistory != 0 ? 1.0f : historyLength;
    // (:568-574) only the signals this kernel was compiled for take part
    historyLength = fminf(historyLength, 1.0f + (DIFF && SPEC ? fmaxf(c.gDiffMaxAccumulatedFrameNum, c.gSpecMaxAccumulatedFrameNum) : (DIFF ? c.gDiffMaxAccumulatedFrameNum : c.gSpecMaxAccumulatedFrameNum)));

    // ---- diffuse (:579-617)
    if (DIFF)
    {
        float diffMaxAccumulatedFrameNum = c.gDiffMaxAccumulatedFrameNum, diffMaxFastAccumulatedFrameNum = c.gDiffMaxFastAccumulatedFrameNum;
        if (c.gHasHistoryConfidence)
        {
            const float conf = LoadR8Unorm(Near(a.diffConfidence), x, y);
            diffMaxAccumulatedFrameNum *= conf;
            diffMaxFastAccumulatedFrameNum *= conf;
        }
        float alpha = SMBReprojectionFound > 0.0f ? fmaxf(1.0f / (diffMaxAccumulatedFrameNum + 1.0f), 1.0f / historyLength) : 1.0f;
        float alphaResponsive = SMBReprojectionFound > 0.0f ? fmaxf(1.0f / (diffMaxFastAccumulatedFrameNum + 1.0f), 1.0f / historyLength) : 1.0f;
        // checkerboarded input: a pixel resolved by the pre-pass accumulates slower (:597-606)
        if (CB && c.gDiffCheckerboard != 2u && CheckerBoard(x, y, c.gFrameIndex) != c.gDiffCheckerboard && historyLength > 1.0f)
        {
            alpha *= 1.0f - c.gCheckerboardResolveAccumSpeed;
            alphaResponsive *= 1.0f - c.gCheckerboardResolveAccumSpeed;
        }
        f4 acc = lerp4(prevDiffSMB, mk4(diffuseIllumination, diffuse2ndMoment), alpha);
        f3 accResponsive = lerp3(prevDiffSMBResponsive, diffuseIllumination, alphaResponsive);
        StoreRGBA16F(a.outDiff, x, y, acc);
        StoreRGBA16F(a.outDiffFast, x, y, mk4(accResponsive, 0.0f));
    }
    StoreR8Unorm(a.outLength, x, y, __fdiv_rn(historyLength, 255.0f));
    if (!SPEC) return;

    // ---- specular (:625-928)
    float specMaxAccumulatedFrameNum = c.gSpecMaxAccumulatedFrameNum, specMaxFastAccumulatedFrameNum = c.gSpecMaxFastAccumulatedFrameNum;
    if (c.gHasHistoryConfidence)
    {
        const float conf = LoadR8Unorm(Near(a.specConfidence), x, y);
        specMaxAccumulatedFrameNum *= conf;
        specMaxFastAccumulatedFrameNum *= conf;
    }
    const float specHistoryFrames = fminf(specMaxAccumulatedFrameNum, historyLength);
    const float specHistoryResponsiveFrames = fminf(specMaxFastAccumulatedFrameNum, historyLength);
    const float hitDist = minHitDist3x3 == kInf ? 0.0f : minHitDist3x3;

    float curvature;
    {
        f2 uvForZeroParallax = c.gOrthoMode == 0.0f ? prevUVSMB : pixelUv;
        f2 zeroUv = GetScreenUv(c.gWorldToClipPrev, prevWorldPos + cameraDelta);
        f2 deltaUv = mk2((uvForZeroParallax.x - zeroUv.x) * fW, (uvForZeroParallax.y - zeroUv.y) * fH);
        float invP = 1.0f / fmaxf(smbParallaxInPixels1, 1.0f / 256.0f);
        deltaUv = deltaUv * invP;
        f3 x10, x01;
        {
            f3 xx = CurWorldPosFromClip(c, (pixelUv.x + c.gRectSizeInv[0]) * 2.0f - 1.0f, pixelUv.y * 2.0f - 1.0f, 1.0f);
            f3 v = c.gOrthoMode == 0.0f ? normalize(-xx) : fwd;
            f3 o = c.gOrthoMode == 0.0f ? mk3(0.0f) : xx;
            x10 = o + v * (dot(currentWorldPos - o, currentNormal) / dot(currentNormal, v));
        }
        {
            f3 xx = CurWorldPosFromClip(c, pixelUv.x * 2.0f - 1.0f, (pixelUv.y + c.gRectSizeInv[1]) * 2.0f - 1.0f, 1.0f);
            f3 v = c.gOrthoMode == 0.0f ? normalize(-xx) : fwd;
            f3 o = c.gOrthoMode == 0.0f ? mk3(0.0f) : xx;
            x01 = o + v * (dot(currentWorldPos - o, currentNormal) / dot(currentNormal, v));
        }
        f2 w = mk2(fabsf(deltaUv.x) + 1.0f / 256.0f, fabsf(deltaUv.y) + 1.0f / 256.0f);
        float wInv = 1.0f / (w.x + w.y);
        w = w * wInv;
        f3 xm = x10 * w.x + x01 * w.y;
        f3 n = normalize(n10 * w.x + n01 * w.y);
        float deltaUvLenFixed = smbParallaxInPixelsMin;
        deltaUvLenFixed *= 1.0f + c.gFramerateScale * Bayer4x4(x, y, c.gFrameIndex);
        // pinned: the snapped uv selects a texel
        float mu = __fadd_rn(pixelUv.x, __fmul_rn(__fmul_rn(deltaUvLenFixed, deltaUv.x), c.gRectSizeInv[0]));
        float mvv = __fadd_rn(pixelUv.y, __fmul_rn(__fmul_rn(deltaUvLenFixed, deltaUv.y), c.gRectSizeInv[1]));
        float fx = floorf(__fmul_rn(mu, fW)), fy = floorf(__fmul_rn(mvv, fH));
        bool inScreen = fx >= 0.0f && fy >= 0.0f && fx < fW && fy < fH;
        if (deltaUvLenFixed > 1.0f && inScreen)
        {
            int ix = (int)fx, iy = (int)fy;
            float zHigh = UnpackViewZ(c, LoadR32F(a.z, ix, iy));
            f3 xHigh = CurWorldPosFromClip(c, (fx + 0.5f) * c.gRectSizeInv[0] * 2.0f - 1.0f, (fy + 0.5f) * c.gRectSizeInv[1] * 2.0f - 1.0f, zHigh);
            f3 nHigh = RX_GUIDE(a, ix, iy).N;
            float zError = fabsf(zHigh - currentLinearZ) / fmaxf(zHigh, currentLinearZ);
            bool cmp = zError < kCurvatureZThreshold;
            n = cmp ? nHigh : n;
            xm = cmp ? xHigh : xm;
        }
        f3 edge = xm - currentWorldPos;
        curvature = dot(n - currentNormal, edge) * PositiveRcp(dot(edge, edge));
    }
    const float hitDistFocused = ThinLens(hitDist, curvature);

    // ================= virtual motion based history (:231-357)
    f4 prevSpecVMB = mk4(0.0f), prevSpecVMBResponsive = mk4(0.0f);
    f3 prevNormalVMB = currentNormal;
    f2 prevUVVMB;
    float prevRoughnessVMB = 0.0f, prevReflectionHitTVMB = c.gDenoisingRange, VMBReprojectionFound;
    const f2 resScalePrev = mk2(c.gRectSizePrev[0] * c.gResourceSizeInvPrev[0], c.gRectSizePrev[1] * c.gResourceSizeInvPrev[1]);
    {
        f3 prevVirtualWorldPos = prevWorldPos + normalize(currentViewVector) * hitDistFocused;
        prevUVVMB = ScreenUvNoKill(c.gWorldToClipPrev, prevVirtualWorldPos);
        if (currentMaterialID == c.gCameraAttachedReflectionMaterialID) prevUVVMB = prevUVSMB;
        const f2 prevPixelPos = mk2(__fmul_rn(prevUVVMB.x, c.gRectSizePrev[0]), __fmul_rn(prevUVVMB.y, c.gRectSizePrev[1]));
        const float tx = __fadd_rn(prevPixelPos.x, -0.5f), ty = __fadd_rn(prevPixelPos.y, -0.5f);
        const float box = floorf(tx), boy = floorf(ty);
        const float bwx = __fadd_rn(tx, -box), bwy = __fadd_rn(ty, -boy);
        const int bx = (int)fmaxf(fminf(box, 1e8f), -1e8f), by = (int)fmaxf(fminf(boy, 1e8f), -1e8f);
        const int zw = a.prevZ.w - 1, zh = a.prevZ.h - 1;
        const f3 cw = currentWorldPos - cameraDelta;
        const float thrBase = disocclusionThreshold * (c.gOrthoMode == 0.0f ? currentLinearZ : 1.0f);
        const float ix0 = (box >= 0.0f && box < c.gRectSizePrev[0]) ? 1.0f : 0.0f, ix1 = (box + 1.0f >= 0.0f && box + 1.0f < c.gRectSizePrev[0]) ? 1.0f : 0.0f;
        const float iy0 = (boy >= 0.0f && boy < c.gRectSizePrev[1]) ? 1.0f : 0.0f, iy1 = (boy + 1.0f >= 0.0f && boy + 1.0f < c.gRectSizePrev[1]) ? 1.0f : 0.0f;
        float tv[4];
#pragma unroll
        for (int k = 0; k < 4; k++)
        {
            int i = k & 1, j = k >> 1;
            int px = clampi(bx + i, 0, zw), py = clampi(by + j, 0, zh);
            float z = UnpackViewZ(c, LoadR32F(a.prevZ, px, py));
            float m = LoadR8Times255(a.prevMaterial, px, py);
            f3 pw = PrevWorldPos(c, bx + i, by + j, z);
            float thr = thrBase * ((i ? ix1 : ix0) * (j ? iy1 : iy0)) - kEps;
            float v = fabsf(dot(cw - pw, currentNormal)) > thr ? 0.0f : 1.0f;
            v *= SameMaterial(currentMaterialID, m, c.gSpecMinMaterial) ? 1.0f : 0.0f;
            tv[k] = v;
        }
        const bool anyValid = tv[0] != 0.0f || tv[1] != 0.0f || tv[2] != 0.0f || tv[3] != 0.0f;
        const bool allValid = tv[0] != 0.0f && tv[1] != 0.0f && tv[2] != 0.0f && tv[3] != 0.0f;
        if (anyValid)
        {
            const float omx = 1.0f - bwx, omy = 1.0f - bwy;
            const f4 bcw = mk4(tv[0] * (omx * omy), tv[1] * (bwx * omy), tv[2] * (omx * bwy), tv[3] * (bwx * bwy));
            const bool useBicubic = SMBReprojectionFound == 2.0f && allValid;
            const CatRomSetup cr = SetupCatRom(prevPixelPos, c.gResourceSizeInvPrev, bcw, useBicubic);
            prevSpecVMB = max4(ResolveCatRom4<false>(cr, a.histSpec), 0.0f);
            prevSpecVMBResponsive = max4(ResolveCatRom4<false>(cr, a.histSpecFast), 0.0f);
            prevReflectionHitTVMB = fmaxf(0.001f, SampleLinear1<false>(a.prevHitDist, prevUVVMB.x * resScalePrev.x, prevUVVMB.y * resScalePrev.y));
            f4 pnr = UnpackPrevNormalRoughness(SampleLinearRGBA8(a.prevNr, prevUVVMB.x * resScalePrev.x, prevUVVMB.y * resScalePrev.y));
            prevNormalVMB = Rotate(c.gWorldPrevToWorld, xyz(pnr));
            prevRoughnessVMB = pnr.w;
        }
        VMBReprojectionFound = allValid ? 1.0f : 0.0f;
    }

    const f4 D = SpecularDominantDirection(currentNormal, V, currentRoughnessModified);
    float virtualHistoryAmount = VMBReprojectionFound * D.w;
    virtualHistoryAmount *= c.gOrthoMode == 0.0f ? 1.0f : 0.75f;
    virtualHistoryAmount *= dot(prevNormalVMB, currentNormalAveraged) > 0.0f ? 1.0f : 0.0f;

    f2 uvDiff = prevUVVMB - prevUVSMB;
    const float uvDiffLengthInPixels = sqrtf(uvDiff.x * fW * (uvDiff.x * fW) + uvDiff.y * fH * (uvDiff.y * fH));
    float tanCurvature = fabsf(curvature * pixelSize);
    tanCurvature *= fmaxf(uvDiffLengthInPixels / fmaxf(NoV, 0.01f), 1.0f);
    const float curvatureAngle = atanf(tanCurvature);

    const float lobeHalfAngle = fmaxf(atanf(RelaxLobeTanHalfAngle(currentRoughnessModified)), kNormalUlp);
    const float normalWeight = EncodingAwareNormalWeight(currentNormal, prevNormalVMB, lobeHalfAngle, curvatureAngle, kNormalUlp, true);
    virtualHistoryAmount *= lerpf(1.0f - saturate(uvDiffLengthInPixels), 1.0f, normalWeight);

    const f2 rrp = RelaxedRoughnessWeightParams(currentRoughness * currentRoughness, c.gRoughnessFraction);
    float virtualRoughnessWeight = NonExpWeight(prevRoughnessVMB * prevRoughnessVMB, rrp.x, rrp.y);
    virtualRoughnessWeight = lerpf(1.0f - saturate(uvDiffLengthInPixels), 1.0f, virtualRoughnessWeight);
    virtualHistoryAmount *= c.gOrthoMode == 0.0f ? virtualRoughnessWeight : 1.0f;
    float specVMBConfidence = virtualRoughnessWeight * 0.9f + 0.1f;

    {
        float rl = rsqrtf(dot(uvDiff, uvDiff));
        uvDiff = uvDiff * rl;
        uvDiff = mk2(uvDiff.x / c.gRectSizePrev[0], uvDiff.y / c.gRectSizePrev[1]);
        uvDiff = uvDiff * (saturate(uvDiffLengthInPixels / 0.1f) + uvDiffLengthInPixels / 2.0f);
    }
    const f2 backUV1 = prevUVVMB + uvDiff, backUV2 = prevUVVMB + uvDiff * 2.0f;
    f4 back1 = UnpackPrevNormalRoughness(SampleLinearRGBA8(a.prevNr, backUV1.x * resScalePrev.x, backUV1.y * resScalePrev.y));
    f4 back2 = UnpackPrevNormalRoughness(SampleLinearRGBA8(a.prevNr, backUV2.x * resScalePrev.x, backUV2.y * resScalePrev.y));
    const f3 bn1 = Rotate(c.gWorldPrevToWorld, xyz(back1)), bn2 = Rotate(c.gWorldPrevToWorld, xyz(back2));
    const bool in1 = backUV1.x > 0.0f && backUV1.y > 0.0f && backUV1.x < 1.0f && backUV1.y < 1.0f;
    const bool in2 = backUV2.x > 0.0f && backUV2.y > 0.0f && backUV2.x < 1.0f && backUV2.y < 1.0f;
    float prevPrevNormalWeight = in1 ? EncodingAwareNormalWeight(prevNormalVMB, bn1, lobeHalfAngle, curvatureAngle * 2.0f, kNormalUlp, true) : 1.0f;
    prevPrevNormalWeight *= in2 ? EncodingAwareNormalWeight(prevNormalVMB, bn2, lobeHalfAngle, curvatureAngle * 3.0f, kNormalUlp, true) : 1.0f;
    virtualHistoryAmount *= 0.33f + 0.67f * prevPrevNormalWeight;
    specVMBConfidence *= 0.33f + 0.67f * prevPrevNormalWeight;
    float rw = NonExpWeight(back1.w * back1.w, rrp.x, rrp.y);
    rw *= NonExpWeight(back2.w * back2.w, rrp.x, rrp.y);
    virtualHistoryAmount *= c.gOrthoMode == 0.0f ? rw * 0.9f + 0.1f : 1.0f;

    const float SMC = SpecMagicCurve(currentRoughnessModified);
    const float hitDistC = lerpf(specularIllumination.w, prevReflectionHitTSMB, SMC);
    const float hitDist1 = ThinLens(hitDistC, curvature), hitDist2 = ThinLens(prevReflectionHitTVMB, curvature);
    const float maxDist = fmaxf(hitDist1, hitDist2);
    const float dHitT = fabsf(hitDist1 - hitDist2);
    const float dHitTMultiplier = lerpf(20.0f, 0.0f, SMC);
    float virtualHistoryHitDistConfidence = 1.0f - saturate(dHitTMultiplier * dHitT / (currentLinearZ + maxDist));
    virtualHistoryHitDistConfidence = lerpf(virtualHistoryHitDistConfidence, 1.0f, SMC);

    {
        f3 virtualWorldPos = XvirtualRx(hitDist, curvature, currentWorldPos, prevWorldPos, currentNormal, V, currentRoughness);
        float virtualWorldPosLength = length(virtualWorldPos);
        float hitDistForTrackingPrev = prevSpecVMBResponsive.w;
        f3 prevVirtualWorldPos = XvirtualRx(hitDistForTrackingPrev, curvature, currentWorldPos, prevWorldPos, currentNormal, V, currentRoughness);
        float virtualWorldPosLengthPrev = length(prevVirtualWorldPos);
        f2 prevUVVMBTest = ScreenUvNoKill(c.gWorldToClipPrev, prevVirtualWorldPos);
        if (currentMaterialID == c.gCameraAttachedReflectionMaterialID) prevUVVMBTest = prevUVSMB;
        float lobeTanHalfAngle = fmaxf(RelaxLobeTanHalfAngle(currentRoughness, 0.6f), 0.5f * c.gRectSizeInv[0]);
        float unproj1 = fminf(hitDist, hitDistForTrackingPrev) / PixelRadiusToWorld(c, 1.0f, fmaxf(virtualWorldPosLength, virtualWorldPosLengthPrev));
        float lobeRadiusInPixels = lobeTanHalfAngle * unproj1;
        float dx = (prevUVVMBTest.x - prevUVVMB.x) * fW, dy = (prevUVVMBTest.y - prevUVVMB.y) * fH;
        float deltaParallaxInPixels = sqrtf(dx * dx + dy * dy);
        virtualHistoryHitDistConfidence *= SmoothStep(lobeRadiusInPixels + 0.25f, 0.0f, deltaParallaxInPixels);
    }

    const float smbFound = SMBReprojectionFound > 0.0f ? 1.0f : 0.0f;
    const float cosVVprev = PinnedDot3(V.x, V.y, V.z, Vprev);
    const float specSMBConfidence = smbFound * SmoothStep01(1.0f - AcosApprox(cosVVprev) / (lobeHalfAngle * NoV / c.gFramerateScale));
    float specSMBAlpha = fmaxf(1.0f - specSMBConfidence, 1.0f / (1.0f + specHistoryFrames));
    float specSMBResponsiveAlpha = fmaxf(specSMBAlpha, 1.0f / (1.0f + specHistoryResponsiveFrames));
    // checkerboarded input (:854-863, :881-887)
    const bool specResolved = CB && c.gSpecCheckerboard != 2u && CheckerBoard(x, y, c.gFrameIndex) != c.gSpecCheckerboard && smbParallaxInPixelsMax < 0.5f;
    if (specResolved)
    {
        const float k = 1.0f - c.gCheckerboardResolveAccumSpeed * smbFound;
        specSMBAlpha *= k;
        specSMBResponsiveAlpha *= k;
    }
    f4 accSMB = mk4(lerp3(xyz(prevSpecSMB), xyz(specularIllumination), specSMBAlpha), lerpf(prevReflectionHitTSMB, specularIllumination.w, fmaxf(specSMBAlpha, 0.1f)));
    float accM2SMB = lerpf(prevSpecSMB.w, specular2ndMoment, specSMBAlpha);
    f3 accSMBResponsive = lerp3(prevSpecSMBResponsive, xyz(specularIllumination), specSMBResponsiveAlpha);

    float specVMBAlpha = fmaxf(1.0f - specVMBConfidence, 1.0f / (1.0f + specHistoryFrames));
    float specVMBResponsiveAlpha = fmaxf(1.0f - specVMBConfidence * virtualHistoryHitDistConfidence, 1.0f / (1.0f + specHistoryResponsiveFrames));
    float specVMBHitTAlpha = fmaxf(1.0f - specVMBConfidence * virtualHistoryHitDistConfidence, 1.0f / (1.0f + specHistoryFrames));
    if (specResolved)
    {
        const float k = 1.0f - c.gCheckerboardResolveAccumSpeed * (VMBReprojectionFound > 0.0f ? 1.0f : 0.0f);
        specVMBAlpha *= k;
        specVMBResponsiveAlpha *= k;
        specVMBHitTAlpha *= k;
    }
    f4 accVMB = mk4(lerp3(xyz(prevSpecVMB), xyz(specularIllumination), specVMBAlpha), lerpf(prevReflectionHitTVMB, specularIllumination.w, fmaxf(specVMBHitTAlpha, 0.1f)));
    float accM2VMB = lerpf(prevSpecVMB.w, specular2ndMoment, specVMBAlpha);
    f3 accVMBResponsive = lerp3(xyz(prevSpecVMBResponsive), xyz(specularIllumination), specVMBResponsiveAlpha);

    virtualHistoryAmount *= saturate(specVMBConfidence / (specSMBConfidence + kEps));
    const float accumulatedReflectionHitT = lerpf(accSMB.w, accVMB.w, virtualHistoryAmount);
    const f3 accSpec = lerp3(xyz(accSMB), xyz(accVMB), virtualHistoryAmount);
    const f3 accSpecResponsive = lerp3(accSMBResponsive, accVMBResponsive, virtualHistoryAmount);
    float accSpec2ndMoment = lerpf(accM2SMB, accM2VMB, virtualHistoryAmount);
    const float specularHistoryConfidence = lerpf(specSMBConfidence, specVMBConfidence, virtualHistoryAmount);
    if (accSpec2ndMoment == 0.0f) accSpec2ndMoment = c.gSpecVarianceBoost * (1.0f - specularHistoryConfidence);

    StoreRGBA16F(a.outSpec, x, y, mk4(accSpec, accSpec2ndMoment));
    StoreRGBA16F(a.outSpecFast, x, y, mk4(accSpecResponsive, hitDist));
    StoreR16F(a.outHitDist, x, y, accumulatedReflectionHitT);
    StoreR8Unorm(a.outConfidence, x, y, specularHistoryConfidence);
}

// =============================================================================================
// History fix (RELAX_HistoryFix.hlsli:10-158)
// =============================================================================================
struct RxHfArgs
{
    RC c;
    Surf tiles, spec, diff, length, nr, z, outSpec, outDiff;
    Surf guide; // decoded guides of the current frame (surf.h PassLaunch::guide)
    int rowBegin, rowEnd;
};
template <bool DIFF, bool SPEC> __global__ void __launch_bounds__(256) RelaxHistoryFixKernel(const __grid_constant__ RxHfArgs a)
{
    const RC& c = a.c;
    const int x = blockIdx.x * 32 + threadIdx.x, y = a.rowBegin + blockIdx.y * 8 + threadIdx.y;
    const int W = c.gRectSize[0], H = c.gRectSize[1];
    if (x >= W || y >= H || y >= a.rowEnd) return;
    if (IsSkyTile(a.tiles, x, y)) return;
    const float centerViewZ = UnpackViewZ(c, LoadR32F(a.z, x, y));
    const float historyLength = LoadR8Times255(a.length, x, y);
    if (centerViewZ > c.gDenoisingRange || historyLength > c.gHistoryFixFrameNum || c.gHistoryFixFrameNum == 1.0f) return;

    // this pass only touches pixels with a young history: the geometry tests run in the oracle's operation order
    const Guide g = DecodeGuidePinned(LoadU32(a.nr, x, y));
    const f3 centerWorldPos = PinnedCurWorldPos(c, x, y, centerViewZ);
    const f3 centerV = -PinnedNormalize(centerWorldPos);
    const float depthThreshold = __fmul_rn(c.gDepthThreshold, c.gOrthoMode == 0.0f ? centerViewZ : 1.0f);
    f4 diffSum = DIFF ? LoadRGBA16F(a.diff, x, y) : mk4(0.0f), specSum = SPEC ? LoadRGBA16F(a.spec, x, y) : mk4(0.0f);
    float diffWSum = 1.0f, specWSum = 1.0f;
    const f2 snwp = NormalWeightParamsAtrous(g.roughness, 5.0f, 1.0f, 0.0f, c.gLobeAngleFraction, c.gSpecLobeAngleSlack);
    const float normalPower = fmaxf(c.gHistoryFixEdgeStoppingNormalPower, 0.01f);
    const float r = floorf(__fadd_rn(__fdiv_rn(c.gHistoryFixBasePixelStride, __fadd_rn(1.0f, historyLength)), 0.5f));
#pragma unroll 1
    for (int j = -2; j <= 2; j++)
#pragma unroll 1
        for (int i = -2; i <= 2; i++)
        {
            if (i == 0 && j == 0) continue;
            int sx = x + (int)((float)i * r), sy = y + (int)((float)j * r);
            if (sx < 0 || sy < 0 || sx >= W || sy >= H) continue; // both weights are zeroed for outside taps
            Guide sg = DecodeGuidePinned(LoadU32(a.nr, sx, sy));
            float sz = UnpackViewZ(c, LoadR32F(a.z, sx, sy));
            f3 sw = PinnedCurWorldPos(c, sx, sy, sz);
            f3 dv = PinnedSub(sw, centerWorldPos);
            float geometryWeight = fabsf(PinnedDot3(dv.x, dv.y, dv.z, g.N)) < depthThreshold ? 1.0f : 0.0f;
            float dw = DIFF ? geometryWeight * powf(fmaxf(0.01f, dot(g.N, sg.N)), normalPower) : 0.0f;
            dw *= SameMaterial(sg.materialID, g.materialID, c.gDiffMinMaterial) ? 1.0f : 0.0f;
            if (DIFF && dw > 1e-4f)
            {
                diffSum = diffSum + LoadRGBA16F(a.diff, sx, sy) * dw;
                diffWSum += dw;
            }
            f3 sampleV = -PinnedNormalize(mk3(__fadd_rn(sw.x, __fmul_rn(c.gRoughnessEdgeStoppingRelaxation, centerWorldPos.x)), __fadd_rn(sw.y, __fmul_rn(c.gRoughnessEdgeStoppingRelaxation, centerWorldPos.y)),
                                                  __fadd_rn(sw.z, __fmul_rn(c.gRoughnessEdgeStoppingRelaxation, centerWorldPos.z))));
            float cosa = fminf(PinnedDot3(g.N.x, g.N.y, g.N.z, sg.N), PinnedDot3(centerV.x, centerV.y, centerV.z, sampleV));
            float swt = geometryWeight * saturate(1.0f - SmoothStep(0.0f, snwp.x, AcosApprox(cosa)) * snwp.y);
            swt *= SameMaterial(sg.materialID, g.materialID, c.gSpecMinMaterial) ? 1.0f : 0.0f;
            if (SPEC && swt > 1e-4f)
            {
                specSum = specSum + LoadRGBA16F(a.spec, sx, sy) * swt;
                specWSum += swt;
            }
        }
    if (DIFF) StoreRGBA16F(a.outDiff, x, y, mk4(diffSum.x / diffWSum, diffSum.y / diffWSum, diffSum.z / diffWSum, diffSum.w / diffWSum));
    if (SPEC) StoreRGBA16F(a.outSpec, x, y, mk4(specSum.x / specWSum, specSum.y / specWSum, specSum.z / specWSum, specSum.w / specWSum));
}

// =============================================================================================
// History clamping + anti-lag (RELAX_HistoryClamping.hlsli:10-364)
// =============================================================================================
struct RxHcArgs
{
    RC c;
    Surf tiles, z, specNoisy, diffNoisy, spec, diff, specFast, diffFast, length;
    Surf outSpec, outDiff, outSpecFast, outDiffFast, outLength;
    int rowBegin, rowEnd;
};
// The 5x5 window of a pixel is shared by up to 25 threads of the CTA: the CTA stages, once, for its (32 + 4) x (8 + 4) texels (clamped
// coordinates, like the reference's Preload, RELAX_HistoryClamping.hlsli:12-60) the responsive history already converted to YCoCg with the
// "inside the denoising range" flag, and the noisy input with its luminance.  The 25 taps are then LDS.128 pairs; the moments are summed
// in the oracle's order (window scan order, individually rounded) because sigma = sqrt(m2 - m1^2) is rounding noise on flat regions.
constexpr int kHcW = 32 + 4, kHcH = 8 + 4;
struct HcTile
{
    float4 fast[kHcH][kHcW];  // {Y, Co, Cg, viewZ < denoisingRange ? 1 : 0}
    float4 noisy[kHcH][kHcW]; // {r, g, b, luminance}
};
__device__ __forceinline__ void StageHcTile(HcTile& tile, const RC& c, const Surf& zSurf, const Surf& inNoisy, const Surf& inFast, int x0, int y0, int tid)
{
    const int W = c.gRectSize[0], H = c.gRectSize[1];
    for (int i = tid; i < kHcW * kHcH; i += 256)
    {
        const int lx = i % kHcW, ly = i / kHcW;
        const int px = clampi(x0 + lx, 0, W - 1), py = clampi(y0 + ly, 0, H - 1);
        // texels beyond the denoising range take no part in the moments: they are staged as zeros (adding +0 is exact) with a zero count
        const bool valid = LoadR32F(zSurf, px, py) < c.gDenoisingRange;
        const f3 sy = valid ? RgbToYCoCg(xyz(LoadRGBA16F(inFast, px, py))) : mk3(0.0f); // exact: power-of-two coefficients
        const f3 n = valid ? xyz(LoadRGBA16F(inNoisy, px, py)) : mk3(0.0f);
        tile.fast[ly][lx] = make_float4(sy.x, sy.y, sy.z, valid ? 1.0f : 0.0f);
        tile.noisy[ly][lx] = make_float4(n.x, n.y, n.z, valid ? PinnedLuma(n) : 0.0f);
    }
}
template <bool IS_SPEC>
__device__ __forceinline__ void ClampSignal(const RC& c, const HcTile& tile, int x, int y, float historyLength, const Surf& inNoisy, const Surf& inSlow, const Surf& inFast,
                                            const Surf& outSlow, const Surf& outFast)
{
    f3 m1 = mk3(0.0f), m2 = mk3(0.0f), noisyM1 = mk3(0.0f);
    float noisyM2 = 0.0f, sum = 0.0f;
    const int cx = threadIdx.x + 2, cy = threadIdx.y + 2;
#pragma unroll
    for (int dx = -2; dx <= 2; dx++)
#pragma unroll
        for (int dy = -2; dy <= 2; dy++)
        {
            const float4 f = tile.fast[cy + dy][cx + dx];
            const float4 nl = tile.noisy[cy + dy][cx + dx];
            const f3 sy = mk3(f.x, f.y, f.z), n = mk3(nl.x, nl.y, nl.z);
            m1 = PinnedAdd(m1, sy);
            m2 = PinnedAdd(m2, mk3(__fmul_rn(sy.x, sy.x), __fmul_rn(sy.y, sy.y), __fmul_rn(sy.z, sy.z)));
            noisyM1 = PinnedAdd(noisyM1, n);
            noisyM2 = __fadd_rn(noisyM2, __fmul_rn(nl.w, nl.w));
            sum += f.w;
        }
    m1 = mk3(__fdiv_rn(m1.x, sum), __fdiv_rn(m1.y, sum), __fdiv_rn(m1.z, sum));
    m2 = mk3(__fdiv_rn(m2.x, sum), __fdiv_rn(m2.y, sum), __fdiv_rn(m2.z, sum));
    noisyM1 = mk3(__fdiv_rn(noisyM1.x, sum), __fdiv_rn(noisyM1.y, sum), __fdiv_rn(noisyM1.z, sum));
    noisyM2 = __fdiv_rn(noisyM2, sum);
    f3 var = mk3(__fadd_rn(m2.x, -__fmul_rn(m1.x, m1.x)), __fadd_rn(m2.y, -__fmul_rn(m1.y, m1.y)), __fadd_rn(m2.z, -__fmul_rn(m1.z, m1.z)));
    f3 sigma = mk3(__fsqrt_rn(fmaxf(0.0f, var.x)), __fsqrt_rn(fmaxf(0.0f, var.y)), __fsqrt_rn(fmaxf(0.0f, var.z)));
    f3 cmin = m1 - sigma * c.gColorBoxSigmaScale, cmax = m1 + sigma * c.gColorBoxSigmaScale;
    const f4 fastCenter = LoadRGBA16F(inFast, x, y);
    const f3 responsiveYCoCg = RgbToYCoCg(xyz(fastCenter));
    cmin = min3(cmin, responsiveYCoCg);
    cmax = max3(cmax, responsiveYCoCg);

    const f4 slow = LoadRGBA16F(inSlow, x, y);
    const f3 slowYCoCg = RgbToYCoCg(xyz(slow));
    f3 clampedYCoCg = slowYCoCg;
    const float maxFast = IS_SPEC ? c.gSpecMaxFastAccumulatedFrameNum : c.gDiffMaxFastAccumulatedFrameNum;
    const float maxSlow = IS_SPEC ? c.gSpecMaxAccumulatedFrameNum : c.gDiffMaxAccumulatedFrameNum;
    if (maxFast < maxSlow) clampedYCoCg = min3(max3(slowYCoCg, cmin), cmax);
    const f3 clamped = YCoCgToRgb(clampedYCoCg);

    f4 outS = mk4(clamped, slow.w);
    const f3 responsiveCenter = YCoCgToRgb(responsiveYCoCg);
    f4 outR = mk4(responsiveCenter, IS_SPEC ? fastCenter.w : 0.0f);
    const bool young = historyLength <= c.gHistoryFixFrameNum;
    if (young)
    {
        if (IS_SPEC) outS = outR;
        else outS = mk4(xyz(outR), outS.w);
    }
    float clampingFactor = (clampedYCoCg.x - slowYCoCg.x) == 0.0f ? 0.0f : saturate((clampedYCoCg.x - slowYCoCg.x) / (responsiveYCoCg.x - slowYCoCg.x));
    if (young) clampingFactor = 1.0f;
    float historyDifferenceL = (IS_SPEC ? 0.33f : 1.0f) * kAntilagAccelScale * c.gHistoryAccelerationAmount * Luma(abs3(responsiveCenter - xyz(slow)));
    historyDifferenceL *= clampingFactor;
    if (young) historyDifferenceL = 0.0f;

    const f3 distToNoisy = noisyM1 - responsiveCenter;
    const float distToNoisyL = Luma(abs3(distToNoisy));
    f3 accel = distToNoisyL == 0.0f ? mk3(0.0f) : mk3(distToNoisy.x * historyDifferenceL / distToNoisyL, distToNoisy.y * historyDifferenceL / distToNoisyL, distToNoisy.z * historyDifferenceL / distToNoisyL);
    const float accelL = Luma(abs3(accel));
    const float accelRatio = accelL == 0.0f ? 0.0f : distToNoisyL / accelL;
    if (accelRatio < 1.0f) accel = accel * accelRatio;
    if (accelRatio <= 0.0f) accel = mk3(0.0f);
    outS = mk4(xyz(outS) + accel, outS.w);
    outR = mk4(xyz(outR) + accel, outR.w);

    const float slowL = Luma(xyz(slow));
    const float noisyL = PinnedLuma(noisyM1);
    const float temporalSigma = c.gHistoryResetTemporalSigmaScale * __fsqrt_rn(fmaxf(0.0f, __fadd_rn(noisyM2, -__fmul_rn(noisyL, noisyL))));
    const float spatialSigma = c.gHistoryResetSpatialSigmaScale * sigma.x;
    float resetAmount = (IS_SPEC ? 0.5f : 1.0f) * c.gHistoryResetAmount * fmaxf(0.0f, fabsf(slowL - noisyL) - spatialSigma - temporalSigma) /
                        (1.0e-6f + fmaxf(slowL, noisyL) + spatialSigma + temporalSigma);
    resetAmount = saturate(resetAmount);
    const f3 noisyCenter = xyz(LoadRGBA16F(inNoisy, x, y));
    outS = mk4(lerp3(xyz(outS), noisyCenter, resetAmount), outS.w);
    outR = mk4(lerp3(xyz(outR), noisyCenter, resetAmount), outR.w);

    const float outL = Luma(xyz(outS));
    outS.w = fmaxf(0.0f, outS.w + (outL * outL - slowL * slowL));
    StoreRGBA16F(outSlow, x, y, outS);
    StoreRGBA16F(outFast, x, y, outR);
}
template <bool DIFF, bool SPEC> __global__ void __launch_bounds__(256) RelaxHistoryClampingKernel(const __grid_constant__ RxHcArgs a)
{
    const RC& c = a.c;
    __shared__ HcTile sTiles[(SPEC ? 1 : 0) + (DIFF ? 1 : 0)]; // specular first
    HcTile& sSpecTile = sTiles[0];
    HcTile& sDiffTile = sTiles[SPEC && DIFF ? 1 : 0];
    const int W = c.gRectSize[0], H = c.gRectSize[1];
    const int x = blockIdx.x * 32 + threadIdx.x, y = a.rowBegin + blockIdx.y * 8 + threadIdx.y;
    const int tid = threadIdx.y * 32 + threadIdx.x;
    const int tileY = min(a.rowBegin + (int)blockIdx.y * 8, H - 1);
    if ((int)blockIdx.x * 32 >= W || a.rowBegin + (int)blockIdx.y * 8 >= H) return; // CTA beyond the rect (uniform)
    if (IsSkyTile(a.tiles, min((int)blockIdx.x * 32, W - 1), tileY) && IsSkyTile(a.tiles, min((int)blockIdx.x * 32 + 31, W - 1), tileY)) return; // both tiles sky (uniform)
    if (SPEC) StageHcTile(sSpecTile, c, a.z, a.specNoisy, a.specFast, (int)blockIdx.x * 32 - 2, a.rowBegin + (int)blockIdx.y * 8 - 2, tid);
    if (DIFF) StageHcTile(sDiffTile, c, a.z, a.diffNoisy, a.diffFast, (int)blockIdx.x * 32 - 2, a.rowBegin + (int)blockIdx.y * 8 - 2, tid);
    __syncthreads();
    if (x >= W || y >= H || y >= a.rowEnd) return;
    if (IsSkyTile(a.tiles, x, y)) return;
    if (!(LoadR32F(a.z, x, y) < c.gDenoisingRange)) return;
    const float historyLength = LoadR8Times255(a.length, x, y);
    if (SPEC) ClampSignal<true>(c, sSpecTile, x, y, historyLength, a.specNoisy, a.spec, a.specFast, a.outSpec, a.outSpecFast);
    if (DIFF) ClampSignal<false>(c, sDiffTile, x, y, historyLength, a.diffNoisy, a.diff, a.diffFast, a.outDiff, a.outDiffFast);
    StoreU8(a.outLength, x, y, LoadU8(a.length, x, y));
}

// =============================================================================================
// Copy (RELAX_Copy.hlsli:11-24) and anti-firefly (RELAX_AntiFirefly.hlsli:11-222): RelaxSettings::enableAntiFirefly
// =============================================================================================
struct RxCopyArgs
{
    Surf inSpec, inDiff, outSpec, outDiff;
    int gridW, gridH; // texels the reference's 8x8 groups cover (stores beyond the texture are dropped)
    int rowBegin, rowEnd;
};
template <bool DIFF, bool SPEC> __global__ void __launch_bounds__(256) RelaxCopyKernel(const __grid_constant__ RxCopyArgs a)
{
    const int x = blockIdx.x * 32 + threadIdx.x, y = a.rowBegin + blockIdx.y * 8 + threadIdx.y;
    if (x >= a.gridW || y >= a.gridH || y >= a.rowEnd || !Inside(SPEC ? a.outSpec : a.outDiff, x, y)) return;
    if (SPEC) *TexelPtrRW<uint2>(a.outSpec, x, y) = __ldg(TexelPtr<uint2>(Near(a.inSpec), x, y));
    if (DIFF) *TexelPtrRW<uint2>(a.outDiff, x, y) = __ldg(TexelPtr<uint2>(Near(a.inDiff), x, y));
}

struct RxAfArgs
{
    RC c;
    Surf tiles, spec, diff, nr, z, outSpec, outDiff;
    int rowBegin, rowEnd;
};
// Cross-bilateral rank-conditioned rank-selection: a centre whose luminance is outside the [min, max] of its same-material 3x3
// neighbours is replaced by that extreme neighbour.  The CTA stages the (32 + 2) x (8 + 2) tile of both signals' luminance and
// colour and the material ids in shared memory once (the reference's Preload, :22-38: clamped coordinates); the 8 neighbours are
// LDS.  Visiting order and strict comparisons are the reference's (ties keep the first extreme met, rows first).
constexpr int kAfW = 32 + 2, kAfH = 8 + 2;
template <bool DIFF, bool SPEC> __global__ void __launch_bounds__(256) RelaxAntiFireflyKernel(const __grid_constant__ RxAfArgs a)
{
    const RC& c = a.c;
    __shared__ uint2 sSpec[kAfH][kAfW], sDiff[kAfH][kAfW];
    __shared__ float sSpecLuma[kAfH][kAfW], sDiffLuma[kAfH][kAfW];
    __shared__ unsigned char sMaterial[kAfH][kAfW];
    const int W = c.gRectSize[0], H = c.gRectSize[1];
    const int x0 = blockIdx.x * 32 - 1, y0 = a.rowBegin + blockIdx.y * 8 - 1;
    const int tid = threadIdx.y * 32 + threadIdx.x;
    const int tileY = min(a.rowBegin + (int)blockIdx.y * 8, H - 1);
    const bool skyTile = IsSkyTile(a.tiles, min((int)blockIdx.x * 32, W - 1), tileY) && IsSkyTile(a.tiles, min((int)blockIdx.x * 32 + 31, W - 1), tileY);
    if (skyTile) return; // both 16x16 tiles this CTA covers are sky: nothing to do (uniform, before any barrier)
    for (int i = tid; i < kAfW * kAfH; i += 256)
    {
        const int lx = i % kAfW, ly = i / kAfW;
        const int px = clampi(x0 + lx, 0, W - 1), py = clampi(y0 + ly, 0, H - 1);
        const uint2 sp = SPEC ? __ldg(TexelPtr<uint2>(a.spec, px, py)) : make_uint2(0u, 0u), df = DIFF ? __ldg(TexelPtr<uint2>(a.diff, px, py)) : make_uint2(0u, 0u);
        sSpec[ly][lx] = sp;
        sDiff[ly][lx] = df;
        // rank selection compares luminances: evaluated in the oracle's operation order, so that near-ties select the same texel
        const f4 sf = UnpackHalf4(sp), dfv = UnpackHalf4(df);
        sSpecLuma[ly][lx] = __fadd_rn(__fadd_rn(__fmul_rn(sf.x, 0.2126f), __fmul_rn(sf.y, 0.7152f)), __fmul_rn(sf.z, 0.0722f));
        sDiffLuma[ly][lx] = __fadd_rn(__fadd_rn(__fmul_rn(dfv.x, 0.2126f), __fmul_rn(dfv.y, 0.7152f)), __fmul_rn(dfv.z, 0.0722f));
        sMaterial[ly][lx] = (unsigned char)(LoadU32(a.nr, px, py) >> 30);
    }
    __syncthreads();
    const int x = blockIdx.x * 32 + threadIdx.x, y = a.rowBegin + blockIdx.y * 8 + threadIdx.y;
    if (x >= W || y >= H || y >= a.rowEnd) return;
    if (IsSkyTile(a.tiles, x, y)) return;
    if (UnpackViewZ(c, LoadR32F(Near(a.z), x, y)) > c.gDenoisingRange) return;

    const int cx = threadIdx.x + 1, cy = threadIdx.y + 1;
    const float centerMaterialID = (float)sMaterial[cy][cx];
    float maxS = -1.0f, minS = 1.0e6f, maxD = -1.0f, minD = 1.0e6f;
    int maxSAt = cy * kAfW + cx, minSAt = maxSAt, maxDAt = maxSAt, minDAt = maxSAt;
#pragma unroll
    for (int yy = -1; yy <= 1; yy++)
#pragma unroll
        for (int xx = -1; xx <= 1; xx++)
        {
            if (xx == 0 && yy == 0) continue;
            if (x + xx < 0 || y + yy < 0 || x + xx >= W || y + yy >= H) continue;
            const int at = (cy + yy) * kAfW + cx + xx;
            const float m = (float)sMaterial[cy + yy][cx + xx];
            if (SameMaterial(m, centerMaterialID, c.gSpecMinMaterial))
            {
                const float l = sSpecLuma[cy + yy][cx + xx];
                if (l > maxS) { maxS = l; maxSAt = at; }
                if (l < minS) { minS = l; minSAt = at; }
            }
            if (SameMaterial(m, centerMaterialID, c.gDiffMinMaterial))
            {
                const float l = sDiffLuma[cy + yy][cx + xx];
                if (l > maxD) { maxD = l; maxDAt = at; }
                if (l < minD) { minD = l; minDAt = at; }
            }
        }
    int sAt = cy * kAfW + cx, dAt = sAt;
    const float ls = sSpecLuma[cy][cx], ld = sDiffLuma[cy][cx];
    if (ls > maxS) sAt = maxSAt;
    if (ls < minS) sAt = minSAt;
    if (ld > maxD) dAt = maxDAt;
    if (ld < minD) dAt = minDAt;
    // colour of the selected texel, second moment of the centre: the .w half is spliced in without a float round trip
    uint2 so = (&sSpec[0][0])[sAt], dn = (&sDiff[0][0])[dAt];
    so.y = (so.y & 0xffffu) | (sSpec[cy][cx].y & 0xffff0000u);
    dn.y = (dn.y & 0xffffu) | (sDiff[cy][cx].y & 0xffff0000u);
    if (SPEC) *TexelPtrRW<uint2>(a.outSpec, x, y) = so;
    if (DIFF) *TexelPtrRW<uint2>(a.outDiff, x, y) = dn;
}

// confidence-driven relaxation of the A-trous edge stopping (RELAX_Atrous.hlsli:55-67, :95-106; RELAX_AtrousSmem.hlsli:189-201, :226-238)
struct ConfidenceRelaxation
{
    float simplifiedSpecularLobeAngleFraction, specularLobeAngleFraction, diffuseLobeAngleFraction;
    float specularLuminanceScale, diffuseLuminanceScale; // multiply the luminance weight exponents
};
template <bool DIFF, bool SPEC, class ARGS>
__device__ __forceinline__ ConfidenceRelaxation RelaxByConfidence(const ARGS& a, int x, int y, float diffuseLobeAngleFraction)
{
    const RC& c = a.c;
    ConfidenceRelaxation r;
    r.simplifiedSpecularLobeAngleFraction = diffuseLobeAngleFraction;
    r.specularLobeAngleFraction = c.gLobeAngleFraction;
    r.diffuseLobeAngleFraction = diffuseLobeAngleFraction;
    r.specularLuminanceScale = r.diffuseLuminanceScale = 1.0f;
    if (c.gHasHistoryConfidence)
    {
        const float sr = saturate(c.gConfidenceDrivenRelaxationMultiplier * (1.0f - (SPEC ? LoadR8Unorm(a.specConfidence, x, y) : 1.0f)));
        float t = saturate(sr * c.gConfidenceDrivenNormalEdgeStoppingRelaxation);
        r.simplifiedSpecularLobeAngleFraction = lerpf(diffuseLobeAngleFraction, 1.0f, t);
        r.specularLobeAngleFraction = lerpf(c.gLobeAngleFraction, 1.0f, t);
        r.specularLuminanceScale = 1.0f - saturate(sr * c.gConfidenceDrivenLuminanceEdgeStoppingRelaxation);
        const float dr = saturate(c.gConfidenceDrivenRelaxationMultiplier * (1.0f - (DIFF ? LoadR8Unorm(a.diffConfidence, x, y) : 1.0f)));
        t = saturate(dr * c.gConfidenceDrivenNormalEdgeStoppingRelaxation);
        r.diffuseLobeAngleFraction = lerpf(diffuseLobeAngleFraction, 1.0f, t);
        r.diffuseLuminanceScale = 1.0f - saturate(dr * c.gConfidenceDrivenLuminanceEdgeStoppingRelaxation);
    }
    return r;
}

// =============================================================================================
// A-trous, first iteration with spatial variance estimation (RELAX_AtrousSmem.hlsli:11-472)
// =============================================================================================
struct RxAtrousArgs
{
    RC c;
    Surf tiles, spec, diff, length, confidence, nr, z, outSpec, outDiff, outNr, outMaterial, outZ;
    Surf specConfidence, diffConfidence; // optional R8_UNORM inputs (confidence-driven relaxation), read only when gHasHistoryConfidence
    Surf guide; // decoded guides of the current frame (surf.h PassLaunch::guide)
    int rowBegin, rowEnd;
    int gridW, gridH; // texels the reference's thread groups cover (first iteration: the previous-frame guides are refreshed for all of them)
};
template <bool DIFF, bool SPEC> __global__ void __launch_bounds__(256) RelaxAtrousSmemKernel(const __grid_constant__ RxAtrousArgs a)
{
    const RC& c = a.c;
    const int x = blockIdx.x * 32 + threadIdx.x, y = a.rowBegin + blockIdx.y * 8 + threadIdx.y;
    const int W = c.gRectSize[0], H = c.gRectSize[1];
    if (y >= a.rowEnd || x >= a.gridW || y >= a.gridH || !Inside(a.outZ, x, y)) return;
    const bool isSky = IsSkyTile(a.tiles, x, y);

    // previous-frame guides are refreshed for every pixel the thread groups cover (:252-266); IN_VIEWZ reads 0 beyond its (rect-origin) view
    const float viewZpacked = Inside(a.z, x, y) ? LoadR32F(a.z, x, y) : 0.0f;
    StoreR32F(a.outZ, x, y, viewZpacked);
    Guide g;
    g.N = mk3(0.0f);
    g.roughness = 0.0f;
    g.materialID = 0.0f;
    if (!isSky) g = RX_GUIDE(a, min(x, W - 1), min(y, H - 1)); // threads of a group that overhang the rect see the clamped texel (the reference's Preload clamps)
    const float centerViewZ = UnpackViewZ(c, viewZpacked);
    f4 nr = mk4(g.N, g.roughness);
    if (centerViewZ > c.gDenoisingRange) nr = mk4(1.0f / 255.0f);
    StoreU32(a.outNr, x, y, PackRGBA8(mk4(__fadd_rn(__fmul_rn(nr.x, 0.5f), 0.5f), __fadd_rn(__fmul_rn(nr.y, 0.5f), 0.5f), __fadd_rn(__fmul_rn(nr.z, 0.5f), 0.5f), nr.w)));
    StoreR8Unorm(a.outMaterial, x, y, __fdiv_rn(g.materialID, 255.0f));

    if (isSky || x >= W || y >= H) return;
    if (centerViewZ > c.gDenoisingRange) return;
    const f3 centerNormal = g.N;
    const float centerRoughness = g.roughness, centerMaterialID = g.materialID;
    const float historyLength = LoadR8Times255(a.length, x, y);

    if (historyLength >= c.gHistoryThreshold)
    {
        // 3x3 gaussian of the moments -> variance (:30-83), fused with the first 3x3 filter (:94-237)
        const f3 centerWorldPos = CurWorldPos(c, x, y, centerViewZ);
        f4 specSum = mk4(0.0f), diffSum = mk4(0.0f);
#pragma unroll
        for (int dx = -1; dx <= 1; dx++)
#pragma unroll
            for (int dy = -1; dy <= 1; dy++)
            {
                int px = clampi(x + dx, 0, W - 1), py = clampi(y + dy, 0, H - 1);
                float k = (dx == 0 ? 0.5f : 0.25f) * (dy == 0 ? 0.5f : 0.25f);
                specSum = specSum + LoadSignal<SPEC>(a.spec, px, py) * k;
                diffSum = diffSum + LoadSignal<DIFF>(a.diff, px, py) * k;
            }
        const float s1 = Luma(xyz(specSum)), d1 = Luma(xyz(diffSum));
        const float centerSpecularVar = fmaxf(0.0f, specSum.w - s1 * s1), centerDiffuseVar = fmaxf(0.0f, diffSum.w - d1 * d1);

        const float centerSpecularLuminance = Luma(xyz(LoadSignal<SPEC>(a.spec, x, y)));
        const float specularPhiLIlluminationInv = 1.0f / fmaxf(1.0e-4f, c.gSpecPhiLuminance * sqrtf(centerSpecularVar));
        const f2 rwp = RoughnessWeightParams(centerRoughness, c.gRoughnessFraction);
        const float specularReprojectionConfidence = (SPEC ? LoadR8Unorm(a.confidence, x, y) : 1.0f);
        const ConfidenceRelaxation cr = RelaxByConfidence<DIFF, SPEC>(a, x, y, c.gLobeAngleFraction);
        const float specularLuminanceWeightRelaxation = lerpf(1.0f, specularReprojectionConfidence, c.gLuminanceEdgeStoppingRelaxation) * cr.specularLuminanceScale;
        const float diffuseNormalWeightParam = NormalWeightParam2(1.0f, cr.diffuseLobeAngleFraction);
        const float simplifiedSpecularNormalWeightParam = NormalWeightParam2(1.0f, cr.simplifiedSpecularLobeAngleFraction);
        const f2 snwp = NormalWeightParamsAtrous(centerRoughness, historyLength, specularReprojectionConfidence, c.gNormalEdgeStoppingRelaxation, cr.specularLobeAngleFraction, c.gSpecLobeAngleSlack);
        const f3 centerV = -normalize(centerWorldPos);
        const float centerDiffuseLuminance = Luma(xyz(LoadSignal<DIFF>(a.diff, x, y)));
        const float diffusePhiLIlluminationInv = 1.0f / fmaxf(1.0e-4f, c.gDiffPhiLuminance * sqrtf(centerDiffuseVar));
        const float depthThreshold = c.gDepthThreshold * (c.gOrthoMode == 0.0f ? centerViewZ : 1.0f);
        float sumWSpecular = 0.0f, sumWDiffuse = 0.0f;
        f4 sumSpecular = mk4(0.0f), sumDiffuse = mk4(0.0f);
#pragma unroll
        for (int cx = -1; cx <= 1; cx++)
#pragma unroll
            for (int cy = -1; cy <= 1; cy++)
            {
                const bool isCenter = cx == 0 && cy == 0;
                const bool isInside = x + cx >= 0 && y + cy >= 0 && x + cx < W && y + cy < H;
                const int px = clampi(x + cx, 0, W - 1), py = clampi(y + cy, 0, H - 1);
                const float kernelW = isInside ? (cx == 0 ? 0.44198f : 0.27901f) * (cy == 0 ? 0.44198f : 0.27901f) : 0.0f;
                const Guide sg = RX_GUIDE(a, px, py);
                const f3 sw = CurWorldPos(c, px, py, UnpackViewZ(c, LoadR32F(a.z, px, py)));
                float geometryW = PlaneDistWeightAtrous(centerWorldPos, centerNormal, sw, depthThreshold) * kernelW;
                const float angles = AcosApprox(dot(centerNormal, sg.N));
                const f3 sampleRay = sw + centerWorldPos * c.gRoughnessEdgeStoppingRelaxation; // sampleV = -normalize(sampleRay)
                const float normalWSimplified = NonExpWeight(angles, diffuseNormalWeightParam, 0.0f);
                const float normalWSpecularSimplified = NonExpWeight(angles, simplifiedSpecularNormalWeightParam, 0.0f);
                const float normalWSpecular = SpecularNormalWeightAtrousRaw(snwp, centerNormal, sg.N, centerV, sampleRay);
                const float roughnessW = NonExpWeight(sg.roughness, rwp.x, rwp.y);
                const f4 ss = LoadSignal<SPEC>(a.spec, px, py);
                float lw = fabsf(centerSpecularLuminance - Luma(xyz(ss))) * specularPhiLIlluminationInv;
                lw = fminf(c.gSpecMaxLuminanceRelativeDifference, lw) * specularLuminanceWeightRelaxation;
                float wSpecular = geometryW * __expf(-lw);
                wSpecular *= c.gRoughnessEdgeStoppingEnabled ? normalWSpecular * roughnessW : normalWSpecularSimplified;
                wSpecular = isCenter ? kernelW : wSpecular;
                wSpecular *= SameMaterial(sg.materialID, centerMaterialID, c.gSpecMinMaterial) ? 1.0f : 0.0f;
                sumWSpecular += wSpecular;
                sumSpecular = sumSpecular + ss * wSpecular;

                const f4 sd = LoadSignal<DIFF>(a.diff, px, py);
                float dlw = fminf(c.gDiffMaxLuminanceRelativeDifference, fabsf(centerDiffuseLuminance - Luma(xyz(sd))) * diffusePhiLIlluminationInv) * cr.diffuseLuminanceScale;
                float wDiffuse = geometryW * normalWSimplified * __expf(-dlw);
                wDiffuse = isCenter ? kernelW : wDiffuse;
                wDiffuse *= SameMaterial(sg.materialID, centerMaterialID, c.gDiffMinMaterial) ? 1.0f : 0.0f;
                sumWDiffuse += wDiffuse;
                sumDiffuse = sumDiffuse + sd * wDiffuse;
            }
        sumWSpecular = fmaxf(sumWSpecular, 1e-6f);
        sumSpecular = mk4(sumSpecular.x / sumWSpecular, sumSpecular.y / sumWSpecular, sumSpecular.z / sumWSpecular, sumSpecular.w / sumWSpecular);
        const float sp1 = Luma(xyz(sumSpecular));
        if (SPEC) StoreRGBA16F(a.outSpec, x, y, mk4(xyz(sumSpecular), fmaxf(0.0f, sumSpecular.w - sp1 * sp1)));
        sumWDiffuse = fmaxf(sumWDiffuse, 1e-6f);
        sumDiffuse = mk4(sumDiffuse.x / sumWDiffuse, sumDiffuse.y / sumWDiffuse, sumDiffuse.z / sumWDiffuse, sumDiffuse.w / sumWDiffuse);
        const float dp1 = Luma(xyz(sumDiffuse));
        if (DIFF) StoreRGBA16F(a.outDiff, x, y, mk4(xyz(sumDiffuse), fmaxf(0.0f, sumDiffuse.w - dp1 * dp1)));
    }
    else
    {
        // short history: 5x5 cross-bilateral estimate of the spatial variance, boosted (:392-470)
        float sumWS = 0.0f, sumS1 = 0.0f, sumS2 = 0.0f, sumWD = 0.0f, sumD1 = 0.0f, sumD2 = 0.0f;
        f3 sumS = mk3(0.0f), sumD = mk3(0.0f);
        const float normalWeightParam = NormalWeightParam2(1.0f, c.gLobeAngleFraction);
#pragma unroll 1
        for (int cx = -2; cx <= 2; cx++)
#pragma unroll 1
            for (int cy = -2; cy <= 2; cy++)
            {
                const int px = clampi(x + cx, 0, W - 1), py = clampi(y + cy, 0, H - 1);
                const Guide sg = RX_GUIDE(a, px, py);
                const float normalW = NonExpWeight(AcosApprox(dot(centerNormal, sg.N)), normalWeightParam, 0.0f);
                const f4 ss = LoadSignal<SPEC>(a.spec, px, py);
                const float specularW = normalW * (SameMaterial(sg.materialID, centerMaterialID, c.gSpecMinMaterial) ? 1.0f : 0.0f);
                sumWS += specularW;
                sumS = sumS + xyz(ss) * specularW;
                sumS1 += Luma(xyz(ss)) * specularW;
                sumS2 += ss.w * specularW;
                const f4 sd = LoadSignal<DIFF>(a.diff, px, py);
                const float diffuseW = normalW * (SameMaterial(sg.materialID, centerMaterialID, c.gDiffMinMaterial) ? 1.0f : 0.0f);
                sumWD += diffuseW;
                sumD = sumD + xyz(sd) * diffuseW;
                sumD1 += Luma(xyz(sd)) * diffuseW;
                sumD2 += sd.w * diffuseW;
            }
        const float boost = fmaxf(1.0f, 4.0f / (historyLength + 1.0f));
        sumWS = fmaxf(sumWS, 1e-6f);
        sumS1 /= sumWS;
        sumS2 /= sumWS;
        if (SPEC) StoreRGBA16F(a.outSpec, x, y, mk4(sumS.x / sumWS, sumS.y / sumWS, sumS.z / sumWS, fmaxf(0.0f, sumS2 - sumS1 * sumS1) * boost));
        sumWD = fmaxf(sumWD, 1e-6f);
        sumD1 /= sumWD;
        sumD2 /= sumWD;
        if (DIFF) StoreRGBA16F(a.outDiff, x, y, mk4(sumD.x / sumWD, sumD.y / sumWD, sumD.z / sumWD, fmaxf(0.0f, sumD2 - sumD1 * sumD1) * boost));
    }
}

// =============================================================================================
// A-trous (RELAX_Atrous.hlsli:11-243)
// =============================================================================================
template <bool DIFF, bool SPEC> __global__ void __launch_bounds__(256) RelaxAtrousKernel(const __grid_constant__ RxAtrousArgs a)
{
    const RC& c = a.c;
    const int x = blockIdx.x * 32 + threadIdx.x, y = a.rowBegin + blockIdx.y * 8 + threadIdx.y;
    const int W = c.gRectSize[0], H = c.gRectSize[1];
    if (x >= W || y >= H || y >= a.rowEnd) return;
    if (IsSkyTile(a.tiles, x, y)) return;
    const float centerViewZ = UnpackViewZ(c, LoadR32F(a.z, x, y));
    if (centerViewZ > c.gDenoisingRange) return;
    const Guide g = RX_GUIDE(a, x, y);
    const f3 centerNormal = g.N;
    const float historyLength = LoadR8Times255(a.length, x, y);
    const int step = (int)c.gStepSize;

    float diffuseLobeAngleFraction = c.gLobeAngleFraction / sqrtf((float)c.gStepSize);
    diffuseLobeAngleFraction = lerpf(0.99f, diffuseLobeAngleFraction, saturate(historyLength / 5.0f));

    const f4 centerSpec = LoadSignal<SPEC>(a.spec, x, y);
    const float centerSpecularLuminance = Luma(xyz(centerSpec));
    const float specularPhiLIlluminationInv = 1.0f / fmaxf(1.0e-4f, c.gSpecPhiLuminance * sqrtf(centerSpec.w));
    const f2 rwp = RoughnessWeightParams(g.roughness, c.gRoughnessFraction);
    const float specularReprojectionConfidence = (SPEC ? LoadR8Unorm(a.confidence, x, y) : 1.0f);
    float specularLuminanceWeightRelaxation = 1.0f;
    if (c.gStepSize <= 4) specularLuminanceWeightRelaxation = lerpf(1.0f, specularReprojectionConfidence, c.gLuminanceEdgeStoppingRelaxation);
    const ConfidenceRelaxation cr = RelaxByConfidence<DIFF, SPEC>(a, x, y, diffuseLobeAngleFraction);
    specularLuminanceWeightRelaxation *= cr.specularLuminanceScale;
    const float normalWeightParam = NormalWeightParam2(1.0f, cr.diffuseLobeAngleFraction);
    const float simplifiedSpecularNormalWeightParam = NormalWeightParam2(1.0f, cr.simplifiedSpecularLobeAngleFraction);
    const f2 snwp = NormalWeightParamsAtrous(g.roughness, historyLength, specularReprojectionConfidence, c.gNormalEdgeStoppingRelaxation, cr.specularLobeAngleFraction, c.gSpecLobeAngleSlack);
    const float w0 = 0.44198f * 0.44198f;
    float sumWSpecular = w0, sumWDiffuse = w0;
    f4 sumSpecular = mk4(centerSpec.x * w0, centerSpec.y * w0, centerSpec.z * w0, centerSpec.w * (w0 * w0));
    const f4 centerDiff = LoadSignal<DIFF>(a.diff, x, y);
    const float centerDiffuseLuminance = Luma(xyz(centerDiff));
    const float diffusePhiLIlluminationInv = 1.0f / fmaxf(1.0e-4f, c.gDiffPhiLuminance * sqrtf(centerDiff.w));
    f4 sumDiffuse = mk4(centerDiff.x * w0, centerDiff.y * w0, centerDiff.z * w0, centerDiff.w * (w0 * w0));

    const f3 centerWorldPos = CurWorldPos(c, x, y, centerViewZ);
    const f3 centerV = -normalize(centerWorldPos);
    const float depthThreshold = c.gDepthThreshold * (c.gOrthoMode == 0.0f ? centerViewZ : 1.0f);

    int offx = 0, offy = 0;
    if (c.gStepSize > 4)
    {
        RngHash rng;
        rng.Initialize(x, y, c.gFrameIndex);
        float r0 = rng.GetFloat(), r1 = rng.GetFloat();
        float half = __fmul_rn((float)c.gStepSize, 0.5f);
        offx = (int)__fmul_rn(half, __fadd_rn(r0, -0.5f));
        offy = (int)__fmul_rn(half, __fadd_rn(r1, -0.5f));
    }
    // Per-tap work is kept to what depends on the tap (these kernels are issue-bound, ~8 taps x 5 iterations per pixel):
    //  * the pixel ray F + R * csx - U * csy is affine in the pixel position: the ray of the centre tap position (x + off) and the
    //    two per-step increments are evaluated once, a tap adds them with compile-time signs (perspective: world position = ray * viewZ);
    //  * the plane distance dot(sw - cw, cn) is viewZ * dot(ray, cn) - dot(cw, cn);
    //  * the tap's view vector is never normalised: dot(v0, -s / |s|) = -dot(v0, s) * rsqrt(dot(s, s));
    //  * viewZ comes with the guide texel (RELAX_ClassifyTiles stores the raw viewZ in its .w), the luminance weights use ex2.approx.
    const bool perspective = c.gOrthoMode == 0.0f;
    const float kx = 2.0f * c.gRectSizeInv[0], ky = 2.0f * c.gRectSizeInv[1];
    const float csx0 = ((float)(x + offx) + 0.5f) * kx - 1.0f, csy0 = ((float)(y + offy) + 0.5f) * ky - 1.0f;
    const f3 R = ld3(c.gFrustumRight), U = ld3(c.gFrustumUp), F = ld3(c.gFrustumForward);
    const f3 d0 = R * csx0 - U * csy0;                     // offset of the ray from the forward axis at the (jittered) centre
    const f3 dX = R * ((float)step * kx), dY = U * (-(float)step * ky); // increments per step in x / y
    const float planeC = dot(centerWorldPos, centerNormal);
    const f3 relaxedCenter = centerWorldPos * c.gRoughnessEdgeStoppingRelaxation;
    const float invSpecAngle = 1.0f / snwp.x;
    const float rwpx = rwp.x * (1.0f / 1023.0f);           // applied to the tap's 10-bit roughness code
    const bool roughnessEdgeStopping = c.gRoughnessEdgeStoppingEnabled != 0;
    const bool compareSpecMaterial = c.gSpecMinMaterial < 3.0f, compareDiffMaterial = c.gDiffMinMaterial < 3.0f; // material ids are 0..3
    const unsigned centerPacked = LoadU32(a.nr, x, y);
    const float centerMaterial = (float)(centerPacked >> 30);
#pragma unroll
    for (int yy = -1; yy <= 1; yy++)
#pragma unroll
        for (int xx = -1; xx <= 1; xx++)
        {
            if (xx == 0 && yy == 0) continue;
            const int px = x + offx + xx * step, py = y + offy + yy * step;
            if ((unsigned)px >= (unsigned)W || (unsigned)py >= (unsigned)H) continue; // geometry weight is zero outside
            const float kernelW = (xx == 0 ? 0.44198f : 0.27901f) * (yy == 0 ? 0.44198f : 0.27901f);
            const float4 q = __ldg(TexelPtr<float4>(a.guide, px, py)); // {N.xyz, raw viewZ}
            const unsigned packed = LoadU32(a.nr, px, py);
            const float sz = fabsf(q.w * c.gViewZScale);
            f3 d = d0;
            if (xx != 0) d = xx > 0 ? d + dX : d - dX;
            if (yy != 0) d = yy > 0 ? d + dY : d - dY;
            const f3 sw = perspective ? (F + d) * sz : F * sz + d;
            float geometryW = fabsf(dot(sw, centerNormal) - planeC) < depthThreshold ? kernelW : 0.0f;
            geometryW = sz < c.gDenoisingRange ? geometryW : 0.0f;
            const float cosn = centerNormal.x * q.x + centerNormal.y * q.y + centerNormal.z * q.z;
            const float angles = AcosApprox(cosn);
            const float normalWSimplified = NonExpWeight(angles, normalWeightParam, 0.0f);
            float wSpecular = 0.0f;
            if (SPEC)
            {
                if (roughnessEdgeStopping)
                {
                    // GetSpecularNormalWeight_ATrous (RELAX_Common.hlsli:147-156) with sampleV = -normalize(sw + relaxation * cw)
                    const f3 sr = sw + relaxedCenter;
                    const float cosa = fminf(cosn, -dot(centerV, sr) * rsqrtf(dot(sr, sr)));
                    const float t = SatMul(AcosApprox(cosa), invSpecAngle);
                    const float normalWSpecular = saturate(1.0f - t * t * fmaf(-2.0f, t, 3.0f) * snwp.y);
                    const float roughnessW = NonExpWeight((float)((packed >> 20) & 1023u), rwpx, rwp.y);
                    wSpecular = geometryW * (normalWSpecular * roughnessW);
                }
                else
                    wSpecular = geometryW * NonExpWeight(angles, simplifiedSpecularNormalWeightParam, 0.0f);
                if (compareSpecMaterial) wSpecular = SameMaterial((float)(packed >> 30), centerMaterial, c.gSpecMinMaterial) ? wSpecular : 0.0f;
            }
            if (SPEC && wSpecular > 1e-4f)
            {
                const f4 ss = LoadSignal<SPEC>(a.spec, px, py);
                float lw = fminf(c.gSpecMaxLuminanceRelativeDifference, fabsf(centerSpecularLuminance - Luma(xyz(ss))) * specularPhiLIlluminationInv);
                lw *= specularLuminanceWeightRelaxation;
                wSpecular *= __expf(-lw); // a weight in (0, 1]
                sumWSpecular += wSpecular;
                sumSpecular = sumSpecular + mk4(ss.x * wSpecular, ss.y * wSpecular, ss.z * wSpecular, ss.w * (wSpecular * wSpecular));
            }
            float wDiffuse = geometryW * normalWSimplified;
            if (compareDiffMaterial) wDiffuse = SameMaterial((float)(packed >> 30), centerMaterial, c.gDiffMinMaterial) ? wDiffuse : 0.0f;
            if (DIFF && wDiffuse > 1e-4f)
            {
                const f4 sd = LoadSignal<DIFF>(a.diff, px, py);
                float lw = fminf(c.gDiffMaxLuminanceRelativeDifference, fabsf(centerDiffuseLuminance - Luma(xyz(sd))) * diffusePhiLIlluminationInv) * cr.diffuseLuminanceScale;
                wDiffuse *= __expf(-lw);
                sumWDiffuse += wDiffuse;
                sumDiffuse = sumDiffuse + mk4(sd.x * wDiffuse, sd.y * wDiffuse, sd.z * wDiffuse, sd.w * (wDiffuse * wDiffuse));
            }
        }
    const float s2 = sumWSpecular * sumWSpecular, d2 = sumWDiffuse * sumWDiffuse;
    if (SPEC) StoreRGBA16F(a.outSpec, x, y, mk4(sumSpecular.x / sumWSpecular, sumSpecular.y / sumWSpecular, sumSpecular.z / sumWSpecular, sumSpecular.w / s2));
    if (DIFF) StoreRGBA16F(a.outDiff, x, y, mk4(sumDiffuse.x / sumWDiffuse, sumDiffuse.y / sumWDiffuse, sumDiffuse.z / sumWDiffuse, sumDiffuse.w / d2));
}
} // namespace

// ---------------------------------------------------------------------------------------------
// RELAX_Diffuse_* / RELAX_Specular_* are the two-signal passes without the other signal's bindings (Source/Denoisers/Relax_Diffuse.hpp,
// Relax_Specular.hpp): the bindings of the absent signal are null surfaces, the kernels are compiled without every access to them.
template <bool DIFF, bool SPEC> static cudaError_t LaunchRelaxSignals(const PassLaunch& p, const RC& c)
{
    const int W = c.gRectSize[0];
    const int rows = p.rowEnd - p.rowBegin;
    const dim3 block(32, 8), grid((W + 31) / 32, (rows + 7) / 8);
    Bindings b(p);
    if (p.kind.pass == Pass::HitDistReconstruction || p.kind.pass == Pass::HitDistReconstruction_5x5)
    {
        RxHitDistArgs a;
        a.c = c;
        a.guide = p.guide;
        a.tiles = b.Next(); a.spec = b.Next(SPEC); a.diff = b.Next(DIFF); a.nr = b.Next(); a.z = b.Next(); a.outSpec = b.Next(SPEC); a.outDiff = b.Next(DIFF);
        if (!b.Complete()) return cudaErrorInvalidValue;
        a.rowBegin = p.rowBegin; a.rowEnd = p.rowEnd;
        if (p.kind.pass == Pass::HitDistReconstruction) NRD_B200_LAUNCH(p, grid, block, a, RelaxHitDistReconstructionKernel<DIFF, SPEC, 1>);
        else NRD_B200_LAUNCH(p, grid, block, a, RelaxHitDistReconstructionKernel<DIFF, SPEC, 2>);
    }
    else if (p.kind.pass == Pass::PrePass)
    {
        RxPrePassArgs a;
        a.c = c;
        a.guide = p.guide;
        a.tiles = b.Next(); a.spec = b.Next(SPEC); a.diff = b.Next(DIFF); a.nr = b.Next(); a.z = b.Next(); a.outSpec = b.Next(SPEC); a.outDiff = b.Next(DIFF);
        if (!b.Complete()) return cudaErrorInvalidValue;
        a.rowBegin = p.rowBegin; a.rowEnd = p.rowEnd;
        const bool checkerboard = (DIFF && c.gDiffCheckerboard != 2u) || (SPEC && c.gSpecCheckerboard != 2u);
        if (checkerboard || p.preloadOnly) NRD_B200_LAUNCH(p, grid, block, a, RelaxPrePassKernel<DIFF, SPEC, true>);
        if (!checkerboard || p.preloadOnly) NRD_B200_LAUNCH(p, grid, block, a, RelaxPrePassKernel<DIFF, SPEC>);
    }
    else if (p.kind.pass == Pass::TemporalAccumulation)
    {
        RxTaArgs a;
        a.c = c;
        a.guide = p.guide;
        a.tiles = b.Next(); a.spec = b.Next(SPEC); a.diff = b.Next(DIFF); a.mv = b.Next(); a.nr = b.Next(); a.z = b.Next();
        a.histSpecFast = b.Next(SPEC); a.histDiffFast = b.Next(DIFF); a.histSpec = b.Next(SPEC); a.histDiff = b.Next(DIFF);
        a.prevNr = b.Next(); a.prevZ = b.Next(); a.prevHitDist = b.Next(SPEC); a.prevLength = b.Next(); a.prevMaterial = b.Next();
        a.specConfidence = b.Next(SPEC); a.diffConfidence = b.Next(DIFF); a.mix = b.Next(); // bound to IN_VIEWZ when absent, never read then
        a.outSpec = b.Next(SPEC); a.outDiff = b.Next(DIFF); a.outSpecFast = b.Next(SPEC); a.outDiffFast = b.Next(DIFF); a.outHitDist = b.Next(SPEC);
        a.outLength = b.Next(); a.outConfidence = b.Next(SPEC);
        if (!b.Complete()) return cudaErrorInvalidValue;
        a.rowBegin = p.rowBegin; a.rowEnd = p.rowEnd;
        const bool checkerboard = (DIFF && c.gDiffCheckerboard != 2u) || (SPEC && c.gSpecCheckerboard != 2u);
        if (checkerboard || p.preloadOnly) NRD_B200_LAUNCH(p, dim3((W + 31) / 32, (rows + 3) / 4), dim3(32, 4), a, RelaxTemporalAccumulationKernel<DIFF, SPEC, true>);
        if (!checkerboard || p.preloadOnly) NRD_B200_LAUNCH(p, dim3((W + 31) / 32, (rows + 3) / 4), dim3(32, 4), a, RelaxTemporalAccumulationKernel<DIFF, SPEC>);
    }
    else if (p.kind.pass == Pass::HistoryFix)
    {
        RxHfArgs a;
        a.c = c;
        a.guide = p.guide;
        a.tiles = b.Next(); a.spec = b.Next(SPEC); a.diff = b.Next(DIFF); a.length = b.Next(); a.nr = b.Next(); a.z = b.Next(); a.outSpec = b.Next(SPEC); a.outDiff = b.Next(DIFF);
        if (!b.Complete()) return cudaErrorInvalidValue;
        a.rowBegin = p.rowBegin; a.rowEnd = p.rowEnd;
        NRD_B200_LAUNCH(p, grid, block, a, RelaxHistoryFixKernel<DIFF, SPEC>);
    }
    else if (p.kind.pass == Pass::HistoryClamping)
    {
        RxHcArgs a;
        a.c = c;
        a.tiles = b.Next(); a.z = b.Next(); a.specNoisy = b.Next(SPEC); a.diffNoisy = b.Next(DIFF); a.spec = b.Next(SPEC); a.diff = b.Next(DIFF);
        a.specFast = b.Next(SPEC); a.diffFast = b.Next(DIFF); a.length = b.Next();
        a.outSpec = b.Next(SPEC); a.outDiff = b.Next(DIFF); a.outSpecFast = b.Next(SPEC); a.outDiffFast = b.Next(DIFF); a.outLength = b.Next();
        if (!b.Complete()) return cudaErrorInvalidValue;
        a.rowBegin = p.rowBegin; a.rowEnd = p.rowEnd;
        NRD_B200_LAUNCH(p, grid, block, a, RelaxHistoryClampingKernel<DIFF, SPEC>);
    }
    else if (p.kind.pass == Pass::Copy)
    {
        RxCopyArgs a;
        a.inSpec = b.Next(SPEC); a.inDiff = b.Next(DIFF); a.outSpec = b.Next(SPEC); a.outDiff = b.Next(DIFF);
        if (!b.Complete()) return cudaErrorInvalidValue;
        a.gridW = p.gridW * 8; a.gridH = p.gridH * 8;
        a.rowBegin = p.rowBegin; a.rowEnd = p.rowEnd;
        NRD_B200_LAUNCH(p, dim3(((SPEC ? a.outSpec.w : a.outDiff.w) + 31) / 32, grid.y), block, a, RelaxCopyKernel<DIFF, SPEC>);
    }
    else if (p.kind.pass == Pass::AntiFirefly)
    {
        RxAfArgs a;
        a.c = c;
        a.tiles = b.Next(); a.spec = b.Next(SPEC); a.diff = b.Next(DIFF); a.nr = b.Next(); a.z = b.Next(); a.outSpec = b.Next(SPEC); a.outDiff = b.Next(DIFF);
        if (!b.Complete()) return cudaErrorInvalidValue;
        a.rowBegin = p.rowBegin; a.rowEnd = p.rowEnd;
        NRD_B200_LAUNCH(p, grid, block, a, RelaxAntiFireflyKernel<DIFF, SPEC>);
    }
    else if (p.kind.pass == Pass::AtrousSmem || p.kind.pass == Pass::Atrous)
    {
        const bool smem = p.kind.pass == Pass::AtrousSmem;
        RxAtrousArgs a;
        a.c = c;
        a.guide = p.guide;
        a.tiles = b.Next(); a.spec = b.Next(SPEC); a.diff = b.Next(DIFF); a.length = b.Next(); a.confidence = b.Next(SPEC); a.nr = b.Next(); a.z = b.Next();
        a.specConfidence = b.Next(SPEC); a.diffConfidence = b.Next(DIFF);
        a.outSpec = b.Next(SPEC); a.outDiff = b.Next(DIFF);
        a.rowBegin = p.rowBegin; a.rowEnd = p.rowEnd;
        if (smem)
        {
            a.outNr = b.Next(); a.outMaterial = b.Next(); a.outZ = b.Next();
            if (!b.Complete()) return cudaErrorInvalidValue;
            a.gridW = p.gridW * 8; a.gridH = p.gridH * 8;
            const int coverW = min(a.gridW, p.preloadOnly ? 32 : a.outZ.w), coverRows = min(p.rowEnd, a.gridH) - p.rowBegin;
            NRD_B200_LAUNCH(p, dim3((coverW + 31) / 32, (max(coverRows, 1) + 7) / 8), block, a, RelaxAtrousSmemKernel<DIFF, SPEC>);
        }
        else
        {
            if (!b.Complete()) return cudaErrorInvalidValue;
            a.outNr = a.outMaterial = a.outZ = a.z;
            NRD_B200_LAUNCH(p, grid, block, a, RelaxAtrousKernel<DIFF, SPEC>);
        }
    }
    else
        return cudaErrorNotSupported;
    return cudaGetLastError();
}

cudaError_t LaunchRelax(const PassLaunch& p)
{
    RC c;
    memset(&c, 0, sizeof(c));
    memcpy(&c, p.constants, p.constantsSize < sizeof(RC) ? p.constantsSize : sizeof(RC));
    if (p.kind.pass == Pass::ClassifyTiles)
    {
        RxTilesArgs a;
        Bindings b(p);
        a.z = b.Next(); a.tiles = b.Next();
        if (!b.Complete()) return cudaErrorInvalidValue;
        a.nr = p.guideNr; a.guide = p.guide; a.buildGuide = p.guideMode == 1 ? 1 : 0;
        a.denoisingRange = c.gDenoisingRange; a.tilesW = p.gridW; a.tilesH = p.gridH;
        int warps = a.tilesW * a.tilesH;
        NRD_B200_LAUNCH(p, (warps * 32 + 255) / 256, 256, a, RelaxClassifyTilesKernel);
        return cudaGetLastError();
    }
    if (p.kind.signals == SIGNAL_DIFFUSE) return LaunchRelaxSignals<true, false>(p, c);
    if (p.kind.signals == SIGNAL_SPECULAR) return LaunchRelaxSignals<false, true>(p, c);
    return LaunchRelaxSignals<true, true>(p, c);
}

#if !defined(NRD_B200_NO_STRIPS)
cudaError_t SetPeerTableRelax(int slot, const PeerTable* table, const cudaStream_t* stream) { return SetPeerTableThisTU(slot, table, stream); }
#endif
} // namespace nrdb200
