// Host-visible launchers of the sm_90a kernels.  Every kernel translation unit is compiled twice (common.cuh): NS = nrdb200 is
// the strip (multi-GPU) build, NS = nrdb200_single the one-GPU build.  The executor calls LaunchPass of one build; LaunchPass
// (dispatch.cu) picks the family launcher from PassLaunch::kind, and the family launcher picks the kernel.
#pragma once
#include "common.cuh"
#include "texel_convert.cuh"

namespace nrdb200
{
cudaError_t LaunchReblurClassifyTiles(const PassLaunch& p);
cudaError_t LaunchReblurHitDistReconstruction(const PassLaunch& p);
cudaError_t LaunchReblurPrePass(const PassLaunch& p);
cudaError_t LaunchReblurTemporalAccumulation(const PassLaunch& p);
cudaError_t LaunchReblurHistoryFix(const PassLaunch& p);
cudaError_t LaunchReblurBlur(const PassLaunch& p);
cudaError_t LaunchReblurPostBlur(const PassLaunch& p);
cudaError_t LaunchReblurTemporalStabilization(const PassLaunch& p);
cudaError_t LaunchSigma(const PassLaunch& p);
cudaError_t LaunchRelax(const PassLaunch& p);
cudaError_t LaunchAux(const PassLaunch& p); // split-screen passes, REFERENCE denoiser
cudaError_t LaunchPass(const PassLaunch& p); // cudaErrorNotSupported: the pass has no kernel
// user textures bound as CUDA arrays (user_arrays.cu): array -> shadow (toShadow) or shadow -> array, every item in one launch
cudaError_t LaunchArrayCopies(const ArrayCopyArgs& a, bool toShadow, cudaStream_t stream);

#if !defined(NRD_B200_NO_STRIPS)
// peer address table of one context slot, replicated into the constant memory of every kernel translation unit.
// stream == nullptr: a host table, copied synchronously; else a device table, copied in order on *stream (common.cuh)
cudaError_t SetPeerTableReblurSpatial(int slot, const PeerTable* table, const cudaStream_t* stream);
cudaError_t SetPeerTableReblurHitDist(int slot, const PeerTable* table, const cudaStream_t* stream);
cudaError_t SetPeerTableReblurTemporal(int slot, const PeerTable* table, const cudaStream_t* stream);
cudaError_t SetPeerTableSigma(int slot, const PeerTable* table, const cudaStream_t* stream);
cudaError_t SetPeerTableRelax(int slot, const PeerTable* table, const cudaStream_t* stream);
cudaError_t SetPeerTableAux(int slot, const PeerTable* table, const cudaStream_t* stream);
cudaError_t SetPeerTableRectOrigin(int slot, const PeerTable* table, const cudaStream_t* stream);
cudaError_t SetPeerTables(int slot, const PeerTable* table, const cudaStream_t* stream = nullptr); // all of the above

// Staged guide inputs under rectOrigin.y != 0 (rect_origin.cu): dst texel (x, y) = src texel (x + dx, y + dy) for x in [x0, x1),
// y in [y0, y1); src is read through the owner lookup, dst rows are held locally.
struct ShiftedCopy
{
    Surf dst, src;
    int x0, x1, y0, y1;
    int bytes; // per texel: 1, 4 or 8
};
constexpr int kMaxShiftedCopies = 8;
struct ShiftedCopyArgs
{
    ShiftedCopy items[kMaxShiftedCopies];
    int n, dx, dy;
};
// pull = false: GatherRectOriginKernel (frame start), true: PullRectOriginKernel (after a pass wrote a staged input)
cudaError_t LaunchShiftedCopies(const ShiftedCopyArgs& a, bool pull, cudaStream_t stream);
cudaError_t PreloadShiftedCopies(); // loads both kernels (see NRD_B200_LAUNCH: nothing may load lazily while a barrier spins)
#endif
} // namespace nrdb200

namespace nrdb200_single
{
cudaError_t LaunchPass(const nrdb200_abi::PassLaunch& p);
cudaError_t LaunchArrayCopies(const nrdb200_abi::ArrayCopyArgs& a, bool toShadow, cudaStream_t stream);
}
