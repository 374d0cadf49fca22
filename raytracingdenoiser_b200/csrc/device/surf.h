// Plain data shared by the executor and both builds of the kernels (one-GPU build and strip build, see common.cuh).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../passes.h"

namespace nrdb200_abi
{
constexpr int kMaxPeers = 8;
constexpr int kMaxPeerSlots = 4;

// Strip geometry of one context slot: (arena of rank r) - (local arena), and the first full-resolution row of every rank's
// strip (start[worldSize] = frame height, unused entries = INT_MAX).  Strips are whole 16-row tiles, not necessarily uniform.
struct PeerTable
{
    long long delta[kMaxPeers];
    int start[kMaxPeers + 1];
    int pad_;
};

// A pitched HBM surface.  On one GPU the whole texture is local.  In strip mode (several GPUs, one horizontal strip
// each) a surface holds its own strip plus `halo` ghost rows above and below, which the owner of those
// rows refreshes after every pass that writes them (arena.cu, GhostPushKernel); a tap that lands outside even the
// ghost rows is loaded straight from the owner's HBM: every context carves its surfaces out of one arena with the same
// layout, so that address is the local address plus (arena of the owner - local arena).  Stores are always local.
struct Surf
{
    uint8_t* base;       // address of texel (0, ly0)
    int pitch;           // bytes per row
    int w, h;            // full (virtual) texture size
    int y0, y1;          // rows owned by this context: [y0, y1)  (the whole texture on one GPU)
    int ly0;             // first row held locally (y0 - halo in strip mode, may be negative)
    unsigned lrows;      // rows held locally
    unsigned stripRows;  // strip mode: rows reserved per strip in this texture's own units (capacity); 0 = whole frame is local
    unsigned rowShift;   // log2 of the texture's downsample factor: full-resolution row = y << rowShift (owner lookup)
    int halo;            // ghost rows on either side, in this texture's own units
    int peerSlot;
};

// Launch bookkeeping handed from the executor to the launchers
struct PassLaunch
{
    PassKind kind;         // the pipeline's pass (scheduler.h PipelineKind): picks the launcher, the kernel and the binding layout
    const void* constants; // host pointer to the dispatch's constant block
    uint32_t constantsSize;
    Surf tex[32];          // bindings in DispatchDesc order
    uint8_t texBytes[32];  // bytes per texel of every binding (passes shared by denoisers with different storage formats look at it)
    uint32_t texNum;
    int gridW, gridH;      // DispatchDesc grid (reference thread-group counts)
    int rowBegin, rowEnd;  // rows this launch must produce, in the pass's own pixel units
    cudaStream_t stream;
    bool preloadOnly;      // do not launch: only make the driver load the kernel this pass maps to (see NRD_B200_LAUNCH)
    // Decoded-guide surface (executor-owned RGBA32F, not part of the DispatchDesc): {N.x, N.y, N.z, viewZ (REBLUR: unpacked |z * gViewZScale|, RELAX: raw)} of the current
    // frame's IN_NORMAL_ROUGHNESS / IN_VIEWZ.  guideMode 1 = this pass writes it (REBLUR ClassifyTiles, the first pass of every
    // frame; guideNr = IN_NORMAL_ROUGHNESS, which that dispatch does not bind itself), 2 = it is complete and the filter passes
    // read it at every tap (REBLUR PrePass / Blur / PostBlur), 0 = not used by this pass.
    Surf guide, guideNr;
    int guideMode;
    // 1024 x float4 {SpecMagicCurve(r), lerp(1, hitDistParams.z, saturate(exp2(hitDistParams.w r^2))), 0.298475 log(39.4115 - 39.0029 r), r}
    // for r = i / 1023: every function of the 10-bit roughness alone, evaluated by the executor with the host libm
    const void* roughnessLut;
};
} // namespace nrdb200_abi
