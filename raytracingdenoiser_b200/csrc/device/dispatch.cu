// The one launch entry point of each build of the kernels (launch.h): pass kind -> family launcher.
#include "launch.h"

namespace nrdb200
{
cudaError_t LaunchPass(const PassLaunch& p)
{
    // A rank without rows (a strip below the rect) launches nothing but still takes part in the barriers -- except for the two
    // passes whose grids do not follow rowBegin / rowEnd, because one GPU writes rows beyond the rect there too:
    //   ClassifyTiles that builds the guide: the tiles of the rect may cover the rank's ghost rows, which it decodes itself (the
    //     guide is never pushed);
    //   SIGMA SmoothTiles: every tile row of the texture, beyond the rect from the clamped tiles of the rect; the bicubic tile
    //     fetch at the rect's bottom edge reads them.
    const bool fullGrid = (p.kind.pass == Pass::ClassifyTiles && p.guideMode == 1) || (p.kind.family == Family::SIGMA && p.kind.pass == Pass::SmoothTiles);
    if (p.rowEnd <= p.rowBegin && !fullGrid) return cudaSuccess;
    if (p.kind.pass == Pass::SplitScreen || p.kind.family == Family::REFERENCE) return LaunchAux(p);
    switch (p.kind.family)
    {
        case Family::SIGMA: return LaunchSigma(p);
        case Family::RELAX: return LaunchRelax(p);
        case Family::REBLUR:
            if (p.kind.pass == Pass::ClassifyTiles) return LaunchReblurClassifyTiles(p);
            // every later pass of the frame reads the decoded guide and the roughness table; the executor provides both
            if (!p.preloadOnly && (p.guideMode != 2 || !p.roughnessLut)) return cudaErrorInvalidValue;
            switch (p.kind.pass)
            {
                case Pass::HitDistReconstruction:
                case Pass::HitDistReconstruction_5x5: return LaunchReblurHitDistReconstruction(p);
                case Pass::PrePass: return LaunchReblurPrePass(p);
                case Pass::TemporalAccumulation: return LaunchReblurTemporalAccumulation(p);
                case Pass::HistoryFix: return LaunchReblurHistoryFix(p);
                case Pass::Blur: return LaunchReblurBlur(p);
                case Pass::PostBlur:
                case Pass::PostBlur_NoTemporalStabilization: return LaunchReblurPostBlur(p);
                case Pass::TemporalStabilization: return LaunchReblurTemporalStabilization(p);
                default: return cudaErrorNotSupported;
            }
        default: return cudaErrorNotSupported; // CLEAR: the executor clears itself
    }
}

#if !defined(NRD_B200_NO_STRIPS)
cudaError_t SetPeerTables(int slot, const PeerTable* table, const cudaStream_t* stream)
{
    cudaError_t e = SetPeerTableReblurSpatial(slot, table, stream);
    if (e == cudaSuccess) e = SetPeerTableReblurHitDist(slot, table, stream);
    if (e == cudaSuccess) e = SetPeerTableReblurTemporal(slot, table, stream);
    if (e == cudaSuccess) e = SetPeerTableSigma(slot, table, stream);
    if (e == cudaSuccess) e = SetPeerTableRelax(slot, table, stream);
    if (e == cudaSuccess) e = SetPeerTableAux(slot, table, stream);
    if (e == cudaSuccess) e = SetPeerTableRectOrigin(slot, table, stream);
    return e;
}
#endif
} // namespace nrdb200
