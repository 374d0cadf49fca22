// User textures bound as CUDA arrays (nrdCudaSetUserTextureArray, e.g. Vulkan / D3D12 images imported with
// cudaImportExternalMemory + cudaExternalMemoryGetMappedMipmappedArray).  The kernels read pitched surfaces, so such a texture
// has a pitched shadow in the kernels' format (executor.cu, ForeignTexture); these kernels move texels between the block-linear
// array and the shadow through surf2Dread / surf2Dwrite, with the channel conversion of ConvertFormatKernel:
//   ArrayToShadowKernel  before the passes: the inputs
//   ShadowToArrayKernel  after them: the user textures the passes wrote
// Every texture of one direction is one item of one launch (blockIdx.z).
#include "launch.h"
#include "texel_convert.cuh"

namespace nrdb200
{
namespace
{
// one texel as the widest access its size allows: a 16-byte texel is one 16-byte load / store
__device__ __forceinline__ uint4 ReadArrayTexel(cudaSurfaceObject_t s, int x, int y, int bytes)
{
    uint4 v = make_uint4(0, 0, 0, 0);
    if (bytes == 16) v = surf2Dread<uint4>(s, x * 16, y);
    else if (bytes == 8)
    {
        const uint2 t = surf2Dread<uint2>(s, x * 8, y);
        v.x = t.x, v.y = t.y;
    }
    else if (bytes == 4) v.x = surf2Dread<unsigned>(s, x * 4, y);
    else if (bytes == 2) v.x = surf2Dread<unsigned short>(s, x * 2, y);
    else v.x = surf2Dread<unsigned char>(s, x, y);
    return v;
}
__device__ __forceinline__ void WriteArrayTexel(cudaSurfaceObject_t s, int x, int y, int bytes, uint4 v)
{
    if (bytes == 16) surf2Dwrite(v, s, x * 16, y);
    else if (bytes == 8) surf2Dwrite(make_uint2(v.x, v.y), s, x * 8, y);
    else if (bytes == 4) surf2Dwrite(v.x, s, x * 4, y);
    else if (bytes == 2) surf2Dwrite((unsigned short)v.x, s, x * 2, y);
    else surf2Dwrite((unsigned char)v.x, s, x, y);
}
__device__ __forceinline__ uint4 ReadShadowTexel(const uint8_t* p, int bytes)
{
    uint4 v = make_uint4(0, 0, 0, 0);
    if (bytes == 16) v = *(const uint4*)p;
    else if (bytes == 8)
    {
        const uint2 t = *(const uint2*)p;
        v.x = t.x, v.y = t.y;
    }
    else if (bytes == 4) v.x = *(const unsigned*)p;
    else if (bytes == 2) v.x = *(const unsigned short*)p;
    else v.x = *p;
    return v;
}
__device__ __forceinline__ void WriteShadowTexel(uint8_t* p, int bytes, uint4 v)
{
    if (bytes == 16) *(uint4*)p = v;
    else if (bytes == 8) *(uint2*)p = make_uint2(v.x, v.y);
    else if (bytes == 4) *(unsigned*)p = v.x;
    else if (bytes == 2) *(unsigned short*)p = (unsigned short)v.x;
    else *p = (unsigned char)v.x;
}

// ConvertFormatKernel's rule: channels the source does not have read 0, extra source channels are dropped; the same format is a copy
__device__ __forceinline__ uint4 ConvertTexel(uint4 v, const TexelFormat& from, const TexelFormat& to)
{
    if (from.channels == to.channels && from.kind == to.kind && from.bytes == to.bytes) return v;
    uint4 out = make_uint4(0, 0, 0, 0);
    const uint8_t* s = (const uint8_t*)&v;
    uint8_t* d = (uint8_t*)&out;
#pragma unroll
    for (int ch = 0; ch < 4; ch++)
        if (ch < to.channels) StoreChannel(d, to.kind, ch, ch < from.channels ? LoadChannel(s, from.kind, ch) : 0.0f);
    return out;
}

// one 32x8 block of texels of item blockIdx.z
template <bool TO_SHADOW> __device__ __forceinline__ void ArrayCopyBody(const ArrayCopyArgs& a)
{
    const ArrayCopy& c = a.items[blockIdx.z];
    const int x = (int)(blockIdx.x * 32 + threadIdx.x), y = (int)(blockIdx.y * 8 + threadIdx.y);
    if (x >= c.width || y >= c.height) return;
    uint8_t* texel = c.shadow + (size_t)y * c.pitch + (size_t)x * c.shadowFormat.bytes;
    if (TO_SHADOW) WriteShadowTexel(texel, c.shadowFormat.bytes, ConvertTexel(ReadArrayTexel(c.array, x, y, c.arrayFormat.bytes), c.arrayFormat, c.shadowFormat));
    else WriteArrayTexel(c.array, x, y, c.arrayFormat.bytes, ConvertTexel(ReadShadowTexel(texel, c.shadowFormat.bytes), c.shadowFormat, c.arrayFormat));
}
} // namespace

__global__ void __launch_bounds__(256) ArrayToShadowKernel(const __grid_constant__ ArrayCopyArgs a) { ArrayCopyBody<true>(a); }
__global__ void __launch_bounds__(256) ShadowToArrayKernel(const __grid_constant__ ArrayCopyArgs a) { ArrayCopyBody<false>(a); }

cudaError_t LaunchArrayCopies(const ArrayCopyArgs& a, bool toShadow, cudaStream_t stream)
{
    int blocksX = 0, blocksY = 0;
    for (int i = 0; i < a.n; i++)
    {
        blocksX = max(blocksX, (a.items[i].width + 31) / 32);
        blocksY = max(blocksY, (a.items[i].height + 7) / 8);
    }
    if (blocksX <= 0 || blocksY <= 0) return cudaSuccess;
    const dim3 grid(blocksX, blocksY, a.n), block(32, 8);
    if (toShadow) ArrayToShadowKernel<<<grid, block, 0, stream>>>(a);
    else ShadowToArrayKernel<<<grid, block, 0, stream>>>(a);
    return cudaGetLastError();
}
} // namespace nrdb200
