// Channel conversion between the formats a user texture may be bound in and the one the kernels read (executor.cu, WiderFormat),
// shared by the executor's pitched conversion (ConvertFormatKernel) and the CUDA-array conversion of both kernel builds
// (user_arrays.cu).
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace nrdb200_abi
{
// kind: 0 = UNORM8, 1 = SFLOAT16, 2 = SFLOAT32
__device__ __forceinline__ float LoadChannel(const uint8_t* texel, int kind, int ch)
{
    if (kind == 0) return (float)texel[ch] / 255.0f;
    if (kind == 1) return __half2float(__ushort_as_half(((const unsigned short*)texel)[ch]));
    return ((const float*)texel)[ch];
}
__device__ __forceinline__ void StoreChannel(uint8_t* texel, int kind, int ch, float v)
{
    if (kind == 0) texel[ch] = (unsigned char)__fadd_rn(__fmul_rn(__saturatef(v), 255.0f), 0.5f); // D3D float -> UNORM
    else if (kind == 1) ((unsigned short*)texel)[ch] = __half_as_ushort(__float2half_rn(v));
    else ((float*)texel)[ch] = v;
}

struct TexelFormat
{
    int channels, kind, bytes; // bytes per texel; channels / kind are those of ConvertibleFormat, or 0 / 0 for a format only copied
};

// A user texture bound as a CUDA array (nrdCudaSetUserTextureArray) and its shadow in the kernels' format
struct ArrayCopy
{
    cudaSurfaceObject_t array; // created at bind time; surface x coordinates are in bytes
    uint8_t* shadow;
    size_t pitch;              // of the shadow
    TexelFormat arrayFormat, shadowFormat;
    int width, height;         // texels converted: the context's resourceSize
};
// every user texture of one direction fits in one launch
constexpr int kMaxArrayCopies = 16;
struct ArrayCopyArgs
{
    ArrayCopy items[kMaxArrayCopies];
    int n;
};
} // namespace nrdb200_abi
