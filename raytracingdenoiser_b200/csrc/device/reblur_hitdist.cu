// REBLUR hit-distance reconstruction (3x3 / 5x5) on sm_90a.
// What has to be computed: reference Shaders/Include/REBLUR_HitDistReconstruction.hlsli:10-155 at the default switches
// (REBLUR_USE_DECOMPRESSED_HIT_DIST_IN_RECONSTRUCTION = 0, not performance mode): a pixel whose ray missed (hit distance 0) takes the
// weighted hit distance of its neighbourhood -- plane-distance weight (strict), gaussian, normal and roughness weights (exponential).
//
// How: a dense stencil, so the CTA stages what all its threads share.  The decoded guides {N.xyz, unpacked viewZ} of tile + halo come from
// the guide surface with ONE TMA bulk tensor copy (cp.async.bulk.tensor.2d -> UTMALDG, completion on an mbarrier) issued by one
// thread while all threads stage the two hit distances and the roughness of the same window with clamped loads; the taps are then
// LDS only.  TMA zero-fills outside the surface where the reference clamps to the rect edge: taps index the tile with clamped
// coordinates, and the clamped texel is always inside the staged box.
#include "reblur_math.cuh"
#include "launch.h"
#include "tma.cuh"

namespace nrdb200
{
using namespace rb;

struct HitDistArgs
{
    ReblurConstants c;
    Surf tiles, nr, inDiff, inSpec, outDiff, outSpec, guide;
    const float4* lut;
    int rowBegin, rowEnd;
    int useTma; // the guide window is staged by TMA (else by clamped loads)
    int perf;   // REBLUR_PERFORMANCE_MODE: no normal / roughness weights (REBLUR_HitDistReconstruction.hlsli:106-119)
};

constexpr int kHdTileW = 32, kHdTileH = 8;

template <bool DIFF, bool SPEC, int BORDER>
__global__ void __launch_bounds__(kHdTileW* kHdTileH) ReblurHitDistReconstructionKernel(const __grid_constant__ HitDistArgs a, const __grid_constant__ CUtensorMap guideMap)
{
    constexpr int BW = kHdTileW + 2 * BORDER, BH = kHdTileH + 2 * BORDER;
    __shared__ __align__(128) float4 sGuide[BH][BW]; // {N.xyz, unpacked viewZ}
    __shared__ float2 sHit[BH][BW];                  // {diffuse, specular} normalised hit distance
    __shared__ float sRough[BH][BW];
    __shared__ __align__(8) uint64_t bar;

    const ReblurConstants& c = a.c;
    const int tid = threadIdx.y * kHdTileW + threadIdx.x;
    const int tileX0 = blockIdx.x * kHdTileW, tileY0 = a.rowBegin + blockIdx.y * kHdTileH;
    const int maxX = c.gRectSizeMinusOne[0], maxY = c.gRectSizeMinusOne[1];

    if (a.useTma)
    {
        if (tid == 0) nrdb200_tma::BarrierInit(&bar);
        __syncthreads();
        // x in 32-bit words, y in rows held locally; negative / beyond-the-edge parts of the box arrive as zeros
        if (tid == 0) nrdb200_tma::LoadTile2D(sGuide, &guideMap, (tileX0 - BORDER) * 4, tileY0 - BORDER - a.guide.ly0, &bar, (uint32_t)sizeof(sGuide));
    }

    // meanwhile: hit distances and roughness of the window, clamped to the rect like the reference's Preload (:13-41)
    for (int i = tid; i < BW * BH; i += kHdTileW * kHdTileH)
    {
        const int lx = i % BW, ly = i / BW;
        const int gx = clampi(tileX0 - BORDER + lx, 0, maxX), gy = clampi(tileY0 - BORDER + ly, 0, maxY);
        float2 h = make_float2(0.0f, 0.0f);
        if (DIFF) h.x = LoadRGBA16F(Near(a.inDiff), gx, gy).w;
        if (SPEC) h.y = LoadRGBA16F(Near(a.inSpec), gx, gy).w;
        sHit[ly][lx] = h;
        if (SPEC) sRough[ly][lx] = (float)((LoadU32(Near(a.nr), gx, gy) >> 20) & 1023u) * (1.0f / 1023.0f);
        if (!a.useTma) sGuide[ly][lx] = __ldg(TexelPtr<float4>(Near(a.guide), gx, gy));
    }
    if (a.useTma) nrdb200_tma::BarrierWait(&bar, 0);
    __syncthreads();

    const int x = tileX0 + threadIdx.x, y = tileY0 + threadIdx.y;
    if (x > maxX || y > maxY || y >= a.rowEnd) return;
    if (LoadU8(Near(a.tiles), x >> 4, y >> 4) != 0) return;

    const int cx = threadIdx.x + BORDER, cy = threadIdx.y + BORDER;
    const float4 g0 = sGuide[cy][cx];
    const float viewZ = g0.w; // the guide holds |viewZ * gViewZScale|
    if (viewZ > c.gDenoisingRange) return;

    const f3 N = mk3(g0.x, g0.y, g0.z);
    const float roughness = SPEC ? __ldg(&a.lut[(LoadU32(Near(a.nr), x, y) >> 20) & 1023u]).w : 1.0f;
    const f2 pixelUv = PixelUv(x, y, c.gRectSizeInv);
    const f3 Xv = ReconstructViewPosition(pixelUv, c.gFrustum, viewZ, c.gOrthoMode);
    const f3 Nv = RotateInverse(c.gViewToWorld, N);
    const float frustumSize = c.gMinRectDimMulUnproject * lerpf(viewZ, 1.0f, fabsf(c.gOrthoMode));
    const float geoA = 1.0f / (c.gPlaneDistSensitivity * frustumSize), geoB = -dot(Nv, Xv) * geoA;
    const f2 rrp = RelaxedRoughnessWeightParams(roughness * roughness, 1.0f);
    const float diffNormalParam = NormalWeightParam(1.0f, 1.0f, 1.0f), specNormalParam = NormalWeightParam(1.0f, 1.0f, roughness);

    const float2 hc = sHit[cy][cx];
    f2 sum = mk2(hc.x != 0.0f ? 1000.0f : 0.0f, hc.y != 0.0f ? 1000.0f : 0.0f);
    f2 acc = mk2(hc.x * sum.x, hc.y * sum.y);
#pragma unroll
    for (int j = -BORDER; j <= BORDER; j++)
#pragma unroll
        for (int i = -BORDER; i <= BORDER; i++)
        {
            if (i == 0 && j == 0) continue;
            // IsInScreenNearest(pixelUv + o * rectSizeInv): the neighbour's centre is on screen iff its integer position is
            if ((unsigned)(x + i) > (unsigned)maxX || (unsigned)(y + j) > (unsigned)maxY) continue;
            const int sx = cx + i, sy = cy + j; // in-rect neighbours are never clamped
            const float4 g = sGuide[sy][sx];
            const float zs = g.w;
            const f2 uv = mk2(pixelUv.x + (float)i * c.gRectSizeInv[0], pixelUv.y + (float)j * c.gRectSizeInv[1]);
            const f3 Xvs = ReconstructViewPosition(uv, c.gFrustum, zs, c.gOrthoMode);
            float w = __expf(-0.66f * 0.25f * (float)(i * i + j * j)); // GetGaussianWeight(length(o) * 0.5)
            w *= NonExpWeight(dot(Nv, Xvs), geoA, geoB);
            f2 ww = mk2(w, w);
            if (!a.perf)
            {
                const float angle = AcosApprox(N.x * g.x + N.y * g.y + N.z * g.z);
                ww = mk2(w * ExpWeight(angle, diffNormalParam, 0.0f), w * ExpWeight(angle, specNormalParam, 0.0f));
                if (SPEC)
                {
                    const float r = sRough[sy][sx];
                    ww.y *= ExpWeight(r * r, rrp.x, rrp.y);
                }
            }
            const float2 h = sHit[sy][sx];
            // Denanify + "valid sample" test: a neighbour takes part iff its weight and its hit distance are non-zero
            if (DIFF && ww.x != 0.0f && h.x != 0.0f)
            {
                acc.x = fmaf(h.x, ww.x, acc.x);
                sum.x += ww.x;
            }
            if (SPEC && ww.y != 0.0f && h.y != 0.0f)
            {
                acc.y = fmaf(h.y, ww.y, acc.y);
                sum.y += ww.y;
            }
        }
    if (DIFF)
    {
        f4 d = LoadRGBA16F(Near(a.inDiff), x, y);
        d.w = acc.x / fmaxf(sum.x, kEps);
        StoreRGBA16F(a.outDiff, x, y, d);
    }
    if (SPEC)
    {
        f4 s = LoadRGBA16F(Near(a.inSpec), x, y);
        s.w = acc.y / fmaxf(sum.y, kEps);
        StoreRGBA16F(a.outSpec, x, y, s);
    }
}

template <bool DIFF, bool SPEC, int BORDER> static cudaError_t LaunchHitDist(const PassLaunch& p)
{
    HitDistArgs a;
    a.c = *(const ReblurConstants*)p.constants;
    Bindings b(p);
    a.tiles = b.Next();
    a.nr = b.Next();
    b.Next(); // IN_VIEWZ: the guide surface carries it
    a.inDiff = b.Next(DIFF);
    a.inSpec = b.Next(SPEC);
    a.outDiff = b.Next(DIFF);
    a.outSpec = b.Next(SPEC);
    if (!b.Complete()) return cudaErrorInvalidValue;
    a.guide = p.guide;
    a.perf = p.kind.perf ? 1 : 0;
    a.lut = (const float4*)p.roughnessLut;
    a.rowBegin = p.rowBegin;
    a.rowEnd = p.rowEnd;
    CUtensorMap map;
    memset(&map, 0, sizeof(map));
    a.useTma = !p.preloadOnly && nrdb200_tma::Enabled() && nrdb200_tma::MakeSurfaceMap(a.guide, 4, kHdTileW + 2 * BORDER, kHdTileH + 2 * BORDER, &map);
    const int W = (int)a.c.gRectSize[0];
    dim3 grid((W + kHdTileW - 1) / kHdTileW, (p.rowEnd - p.rowBegin + kHdTileH - 1) / kHdTileH), block(kHdTileW, kHdTileH);
    if (p.preloadOnly)
    {
        cudaFuncAttributes fa;
        return cudaFuncGetAttributes(&fa, ReblurHitDistReconstructionKernel<DIFF, SPEC, BORDER>);
    }
    ReblurHitDistReconstructionKernel<DIFF, SPEC, BORDER><<<grid, block, 0, p.stream>>>(a, map);
    return cudaGetLastError();
}

cudaError_t LaunchReblurHitDistReconstruction(const PassLaunch& p)
{
    const bool is5x5 = p.kind.pass == Pass::HitDistReconstruction_5x5;
    if (p.kind.signals == SIGNAL_DIFFUSE) return is5x5 ? LaunchHitDist<true, false, 2>(p) : LaunchHitDist<true, false, 1>(p);
    if (p.kind.signals == SIGNAL_SPECULAR) return is5x5 ? LaunchHitDist<false, true, 2>(p) : LaunchHitDist<false, true, 1>(p);
    return is5x5 ? LaunchHitDist<true, true, 2>(p) : LaunchHitDist<true, true, 1>(p);
}

#if !defined(NRD_B200_NO_STRIPS)
cudaError_t SetPeerTableReblurHitDist(int slot, const PeerTable* table, const cudaStream_t* stream) { return SetPeerTableThisTU(slot, table, stream); }
#endif
} // namespace nrdb200
