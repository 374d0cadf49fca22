// Staged guide inputs of connected strips under rectOrigin.y != 0 (executor.cu, StagesInputs).  A guide input is read at
// rectOrigin + pixel (WithRectOrigin); shifted by whole rows, a strip's own and ghost rows would hold rows of other strips, and
// the kernels' Near() loads (common.cuh) would read them as local.  Instead each rank keeps a copy of every such input in the
// kernels' layout -- view row y, column x = resource row y + oy, column x + ox -- which the passes bind with origin 0:
//   GatherRectOriginKernel  frame start: fills the copy's own and ghost rows, reading the inputs through the owner lookup
//   PullRectOriginKernel    after a pass that wrote a staged input (REBLUR TemporalStabilization patches IN_MV): each rank copies
//                           its own rows of the input back from the staged view, so the application sees what one GPU writes
// Strip build only: a one-GPU context never stages.
#include "launch.h"

#if !defined(NRD_B200_NO_STRIPS)
namespace nrdb200
{
namespace
{
template <class T> __device__ __forceinline__ void CopyTexel(const ShiftedCopy& c, int x, int y, int dx, int dy)
{
    *TexelPtrRW<T>(c.dst, x, y) = __ldg(TexelPtr<T>(c.src, x + dx, y + dy));
}

// one 32x8 block of texels of copy blockIdx.z
__device__ __forceinline__ void ShiftedCopyBody(const ShiftedCopyArgs& a)
{
    const ShiftedCopy& c = a.items[blockIdx.z];
    const int x = c.x0 + (int)(blockIdx.x * 32 + threadIdx.x), y = c.y0 + (int)(blockIdx.y * 8 + threadIdx.y);
    if (x >= c.x1 || y >= c.y1) return;
    if (c.bytes == 8) CopyTexel<uint2>(c, x, y, a.dx, a.dy);
    else if (c.bytes == 4) CopyTexel<unsigned>(c, x, y, a.dx, a.dy);
    else CopyTexel<unsigned char>(c, x, y, a.dx, a.dy);
}
} // namespace

__global__ void __launch_bounds__(256) GatherRectOriginKernel(const __grid_constant__ ShiftedCopyArgs a) { ShiftedCopyBody(a); }
__global__ void __launch_bounds__(256) PullRectOriginKernel(const __grid_constant__ ShiftedCopyArgs a) { ShiftedCopyBody(a); }

cudaError_t LaunchShiftedCopies(const ShiftedCopyArgs& a, bool pull, cudaStream_t stream)
{
    int blocksX = 0, blocksY = 0;
    for (int i = 0; i < a.n; i++)
    {
        blocksX = max(blocksX, (a.items[i].x1 - a.items[i].x0 + 31) / 32);
        blocksY = max(blocksY, (a.items[i].y1 - a.items[i].y0 + 7) / 8);
    }
    if (blocksX <= 0 || blocksY <= 0) return cudaSuccess; // nothing of the view lies in this rank's rows
    const dim3 grid(blocksX, blocksY, a.n), block(32, 8);
    if (pull) PullRectOriginKernel<<<grid, block, 0, stream>>>(a);
    else GatherRectOriginKernel<<<grid, block, 0, stream>>>(a);
    return cudaGetLastError();
}

cudaError_t PreloadShiftedCopies()
{
    cudaFuncAttributes fa;
    cudaError_t e = cudaFuncGetAttributes(&fa, GatherRectOriginKernel);
    return e == cudaSuccess ? cudaFuncGetAttributes(&fa, PullRectOriginKernel) : e;
}

cudaError_t SetPeerTableRectOrigin(int slot, const PeerTable* table, const cudaStream_t* stream) { return SetPeerTableThisTU(slot, table, stream); }
} // namespace nrdb200
#endif
