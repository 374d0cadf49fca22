// nrd_b200.h -- the drop-in boundary of the H100-native denoiser.
//
// Part 1 restates, layout-for-layout, the C ABI that the reference library exports
// (reference: Include/NRD.h:51-70, Include/NRDDescs.h:20-512, Include/NRDSettings.h:20-462,
// NRD v4.14.0).  An application compiled against the reference headers can link against
// libnrd_b200.so unchanged: symbol names (extern "C", so the nrd:: namespace does not
// mangle), enum values, struct member order/sizes and default settings are identical.
// Part 2 declares the CUDA executor that takes the place of the reference's optional
// Integration/NRDIntegration.hpp layer (which needs the external NRI RHI): it owns the
// pool textures in HBM and launches one sm_90a kernel per DispatchDesc.
//
// This file is written from the interface description, not copied: enumerators are kept in
// X-macro lists so that the name tables, the format tables and the python binding are all
// generated from one place.
#pragma once

#include <cstddef>
#include <cstdint>

#define NRD_VERSION_MAJOR 4
#define NRD_VERSION_MINOR 14
#define NRD_VERSION_BUILD 0
#define NRD_VERSION_DATE "19 February 2025"

#if defined(_WIN32)
#  define NRD_CALL __stdcall
#else
#  define NRD_CALL
#endif
#ifndef NRD_API
#  define NRD_API extern "C" __attribute__((visibility("default")))
#endif

// ---------------------------------------------------------------------------------------------
// Enumerator lists (order == numeric value, reference: NRDDescs.h:37-332)
// ---------------------------------------------------------------------------------------------
#define NRD_B200_RESOURCE_TYPES(X)                                                            \
    X(IN_MV) X(IN_NORMAL_ROUGHNESS) X(IN_VIEWZ) X(IN_DIFF_CONFIDENCE) X(IN_SPEC_CONFIDENCE)    \
    X(IN_DISOCCLUSION_THRESHOLD_MIX) X(IN_BASECOLOR_METALNESS) X(IN_DIFF_RADIANCE_HITDIST)    \
    X(IN_SPEC_RADIANCE_HITDIST) X(IN_DIFF_HITDIST) X(IN_SPEC_HITDIST)                          \
    X(IN_DIFF_DIRECTION_HITDIST) X(IN_DIFF_SH0) X(IN_DIFF_SH1) X(IN_SPEC_SH0) X(IN_SPEC_SH1)   \
    X(IN_PENUMBRA) X(IN_TRANSLUCENCY) X(IN_SIGNAL) X(OUT_DIFF_RADIANCE_HITDIST)                \
    X(OUT_SPEC_RADIANCE_HITDIST) X(OUT_DIFF_SH0) X(OUT_DIFF_SH1) X(OUT_SPEC_SH0)               \
    X(OUT_SPEC_SH1) X(OUT_DIFF_HITDIST) X(OUT_SPEC_HITDIST) X(OUT_DIFF_DIRECTION_HITDIST)      \
    X(OUT_SHADOW_TRANSLUCENCY) X(OUT_SIGNAL) X(OUT_VALIDATION) X(TRANSIENT_POOL)               \
    X(PERMANENT_POOL)

#define NRD_B200_DENOISERS(X)                                                                 \
    X(REBLUR_DIFFUSE) X(REBLUR_DIFFUSE_OCCLUSION) X(REBLUR_DIFFUSE_SH) X(REBLUR_SPECULAR)      \
    X(REBLUR_SPECULAR_OCCLUSION) X(REBLUR_SPECULAR_SH) X(REBLUR_DIFFUSE_SPECULAR)              \
    X(REBLUR_DIFFUSE_SPECULAR_OCCLUSION) X(REBLUR_DIFFUSE_SPECULAR_SH)                         \
    X(REBLUR_DIFFUSE_DIRECTIONAL_OCCLUSION) X(RELAX_DIFFUSE) X(RELAX_DIFFUSE_SH)               \
    X(RELAX_SPECULAR) X(RELAX_SPECULAR_SH) X(RELAX_DIFFUSE_SPECULAR)                           \
    X(RELAX_DIFFUSE_SPECULAR_SH) X(SIGMA_SHADOW) X(SIGMA_SHADOW_TRANSLUCENCY) X(REFERENCE)

// X(name, bytes per texel, is integer format)
#define NRD_B200_FORMATS(X)                                                                   \
    X(R8_UNORM, 1, 0) X(R8_SNORM, 1, 0) X(R8_UINT, 1, 1) X(R8_SINT, 1, 0)                      \
    X(RG8_UNORM, 2, 0) X(RG8_SNORM, 2, 0) X(RG8_UINT, 2, 1) X(RG8_SINT, 2, 0)                  \
    X(RGBA8_UNORM, 4, 0) X(RGBA8_SNORM, 4, 0) X(RGBA8_UINT, 4, 1) X(RGBA8_SINT, 4, 0)          \
    X(RGBA8_SRGB, 4, 0)                                                                       \
    X(R16_UNORM, 2, 0) X(R16_SNORM, 2, 0) X(R16_UINT, 2, 1) X(R16_SINT, 2, 0)                  \
    X(R16_SFLOAT, 2, 0)                                                                       \
    X(RG16_UNORM, 4, 0) X(RG16_SNORM, 4, 0) X(RG16_UINT, 4, 1) X(RG16_SINT, 4, 0)              \
    X(RG16_SFLOAT, 4, 0)                                                                      \
    X(RGBA16_UNORM, 8, 0) X(RGBA16_SNORM, 8, 0) X(RGBA16_UINT, 8, 1) X(RGBA16_SINT, 8, 0)      \
    X(RGBA16_SFLOAT, 8, 0)                                                                    \
    X(R32_UINT, 4, 1) X(R32_SINT, 4, 0) X(R32_SFLOAT, 4, 0)                                    \
    X(RG32_UINT, 8, 1) X(RG32_SINT, 8, 0) X(RG32_SFLOAT, 8, 0)                                 \
    X(RGB32_UINT, 12, 1) X(RGB32_SINT, 12, 0) X(RGB32_SFLOAT, 12, 0)                           \
    X(RGBA32_UINT, 16, 1) X(RGBA32_SINT, 16, 0) X(RGBA32_SFLOAT, 16, 0)                        \
    X(R10_G10_B10_A2_UNORM, 4, 0) X(R10_G10_B10_A2_UINT, 4, 1) X(R11_G11_B10_UFLOAT, 4, 0)     \
    X(R9_G9_B9_E5_UFLOAT, 4, 0)

namespace nrd
{
typedef uint32_t Identifier;
struct Instance; // opaque

enum class Result : uint32_t { SUCCESS, FAILURE, INVALID_ARGUMENT, UNSUPPORTED, NON_UNIQUE_IDENTIFIER, MAX_NUM };

#define NRD_B200_ENUMERATOR(name, ...) name,
enum class ResourceType : uint32_t { NRD_B200_RESOURCE_TYPES(NRD_B200_ENUMERATOR) MAX_NUM };
enum class Denoiser : uint32_t { NRD_B200_DENOISERS(NRD_B200_ENUMERATOR) MAX_NUM };
enum class Format : uint32_t { NRD_B200_FORMATS(NRD_B200_ENUMERATOR) MAX_NUM };
#undef NRD_B200_ENUMERATOR

enum class DescriptorType : uint32_t { TEXTURE, STORAGE_TEXTURE, MAX_NUM };
enum class Sampler : uint32_t { NEAREST_CLAMP, LINEAR_CLAMP, MAX_NUM };
enum class NormalEncoding : uint8_t { RGBA8_UNORM, RGBA8_SNORM, R10_G10_B10_A2_UNORM, RGBA16_UNORM, RGBA16_SNORM, MAX_NUM };
enum class RoughnessEncoding : uint8_t { SQ_LINEAR, LINEAR, SQRT_LINEAR, MAX_NUM };
// Checkerboarded noisy inputs (NRDSettings.h CheckerboardMode): a signal is traced for every other pixel only -- the pixels with
// ((x ^ y ^ frameIndex) & 1) == parity -- and stored packed, pixel x at column x >> 1 of IN_DIFF_* / IN_SPEC_* (left half of the
// texture).  BLACK: diffuse on parity 0, specular on parity 1; WHITE: the opposite.  Implemented for REBLUR and RELAX.
enum class CheckerboardMode : uint8_t { OFF, BLACK, WHITE, MAX_NUM };
enum class AccumulationMode : uint8_t { CONTINUE, RESTART, CLEAR_AND_RESTART, MAX_NUM };
enum class HitDistanceReconstructionMode : uint8_t { OFF, AREA_3X3, AREA_5X5, MAX_NUM };

// ---- descs (reference: NRDDescs.h:372-512) ---------------------------------------------------
struct AllocationCallbacks
{
    void* (*Allocate)(void* userArg, size_t size, size_t alignment);
    void* (*Reallocate)(void* userArg, void* memory, size_t size, size_t alignment);
    void (*Free)(void* userArg, void* memory);
    void* userArg;
};

struct SPIRVBindingOffsets { uint32_t samplerOffset, textureOffset, constantBufferOffset, storageTextureAndBufferOffset; };

struct LibraryDesc
{
    SPIRVBindingOffsets spirvBindingOffsets;
    const Denoiser* supportedDenoisers;
    uint32_t supportedDenoisersNum;
    uint8_t versionMajor, versionMinor, versionBuild;
    NormalEncoding normalEncoding;
    RoughnessEncoding roughnessEncoding;
};

struct DenoiserDesc { Identifier identifier; Denoiser denoiser; };

struct InstanceCreationDesc
{
    AllocationCallbacks allocationCallbacks;
    const DenoiserDesc* denoisers;
    uint32_t denoisersNum;
};

struct TextureDesc { Format format; uint16_t downsampleFactor; };
struct ResourceDesc { DescriptorType descriptorType; ResourceType type; uint16_t indexInPool; };
struct ResourceRangeDesc { DescriptorType descriptorType; uint32_t baseRegisterIndex; uint32_t descriptorsNum; };
struct ComputeShaderDesc { const void* bytecode; uint64_t size; };

struct PipelineDesc
{
    ComputeShaderDesc computeShaderDXBC;  // always {nullptr, 0}: there is no HLSL bytecode in this build
    ComputeShaderDesc computeShaderDXIL;
    ComputeShaderDesc computeShaderSPIRV;
    const char* shaderFileName;           // reference pass name, e.g. "REBLUR_DiffuseSpecular_Blur.cs"
    const char* shaderEntryPointName;
    const ResourceRangeDesc* resourceRanges;
    uint32_t resourceRangesNum;
    bool hasConstantData;
};

struct DescriptorPoolDesc { uint32_t setsMaxNum, constantBuffersMaxNum, samplersMaxNum, texturesMaxNum, storageTexturesMaxNum; };

struct InstanceDesc
{
    uint32_t constantBufferMaxDataSize;
    uint32_t constantBufferSpaceIndex;
    uint32_t constantBufferRegisterIndex;
    const Sampler* samplers;
    uint32_t samplersNum;
    uint32_t samplersSpaceIndex;
    uint32_t samplersBaseRegisterIndex;
    const PipelineDesc* pipelines;
    uint32_t pipelinesNum;
    uint32_t resourcesSpaceIndex;
    const TextureDesc* permanentPool;
    uint32_t permanentPoolSize;
    const TextureDesc* transientPool;
    uint32_t transientPoolSize;
    DescriptorPoolDesc descriptorPoolDesc;
};

struct DispatchDesc
{
    const char* name;
    Identifier identifier;
    const ResourceDesc* resources;   // all TEXTURE inputs first, then all STORAGE_TEXTURE outputs
    uint32_t resourcesNum;
    const uint8_t* constantBufferData;
    uint32_t constantBufferDataSize;
    bool constantBufferDataMatchesPreviousDispatch;
    uint16_t pipelineIndex;
    uint16_t gridWidth;
    uint16_t gridHeight;
};

// ---- settings (reference: NRDSettings.h:88-448; same defaults) --------------------------------
inline uint32_t GetMaxAccumulatedFrameNum(float accumulationTime, float fps) { return (uint32_t)(accumulationTime * fps); }

struct CommonSettings
{
    float viewToClipMatrix[16] = {};          // column-major, column vectors, non-jittered
    float viewToClipMatrixPrev[16] = {};
    float worldToViewMatrix[16] = {};
    float worldToViewMatrixPrev[16] = {};
    float worldPrevToWorldMatrix[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
    float motionVectorScale[3] = {1.0f, 1.0f, 0.0f};
    float cameraJitter[2] = {};
    float cameraJitterPrev[2] = {};
    uint16_t resourceSize[2] = {};
    uint16_t resourceSizePrev[2] = {};
    uint16_t rectSize[2] = {};
    uint16_t rectSizePrev[2] = {};
    float viewZScale = 1.0f;
    float timeDeltaBetweenFrames = 0.0f;      // ms; 0 = wall clock (non-deterministic)
    float denoisingRange = 500000.0f;
    float disocclusionThreshold = 0.01f;
    float disocclusionThresholdAlternate = 0.05f;
    float cameraAttachedReflectionMaterialID = 999.0f;
    float strandMaterialID = 999.0f;
    float strandThickness = 80e-6f;
    float splitScreen = 0.0f;
    uint16_t printfAt[2] = {9999, 9999};
    float debug = 0.0f;
    uint32_t rectOrigin[2] = {};
    uint32_t frameIndex = 0;
    AccumulationMode accumulationMode = AccumulationMode::CONTINUE;
    bool isMotionVectorInWorldSpace = false;
    bool isHistoryConfidenceAvailable = false;
    bool isDisocclusionThresholdMixAvailable = false;
    bool isBaseColorMetalnessAvailable = false;
    bool enableValidation = false;
};

const uint32_t REBLUR_MAX_HISTORY_FRAME_NUM = 63;
const float REBLUR_DEFAULT_ACCUMULATION_TIME = 0.5f;

struct HitDistanceParameters { float A = 3.0f, B = 0.1f, C = 20.0f, D = -25.0f; };
struct ReblurAntilagSettings { float luminanceSigmaScale = 4.0f; float luminanceSensitivity = 3.0f; };

struct ReblurSettings
{
    HitDistanceParameters hitDistanceParameters = {};
    ReblurAntilagSettings antilagSettings = {};
    uint32_t maxAccumulatedFrameNum = 30;
    uint32_t maxFastAccumulatedFrameNum = 6;
    uint32_t maxStabilizedFrameNum = REBLUR_MAX_HISTORY_FRAME_NUM;
    uint32_t maxStabilizedFrameNumForHitDistance = REBLUR_MAX_HISTORY_FRAME_NUM;
    uint32_t historyFixFrameNum = 3;
    uint32_t historyFixBasePixelStride = 14;
    float diffusePrepassBlurRadius = 30.0f;
    float specularPrepassBlurRadius = 50.0f;
    float minHitDistanceWeight = 0.1f;
    float minBlurRadius = 1.0f;
    float maxBlurRadius = 30.0f;
    float lobeAngleFraction = 0.15f;
    float roughnessFraction = 0.15f;
    float responsiveAccumulationRoughnessThreshold = 0.0f;
    float planeDistanceSensitivity = 0.02f;
    float specularProbabilityThresholdsForMvModification[2] = {0.5f, 0.9f};
    float fireflySuppressorMinRelativeScale = 2.0f;
    CheckerboardMode checkerboardMode = CheckerboardMode::OFF;
    HitDistanceReconstructionMode hitDistanceReconstructionMode = HitDistanceReconstructionMode::OFF;
    bool enableAntiFirefly = false;
    bool enablePerformanceMode = false;
    float minMaterialForDiffuse = 4.0f;
    float minMaterialForSpecular = 4.0f;
    bool usePrepassOnlyForSpecularMotionEstimation = false;
};

const uint32_t RELAX_MAX_HISTORY_FRAME_NUM = 255;
const float RELAX_DEFAULT_ACCUMULATION_TIME = 0.5f;

struct RelaxAntilagSettings
{
    float accelerationAmount = 0.3f;
    float spatialSigmaScale = 4.5f;
    float temporalSigmaScale = 0.5f;
    float resetAmount = 0.5f;
};

struct RelaxSettings
{
    RelaxAntilagSettings antilagSettings = {};
    uint32_t diffuseMaxAccumulatedFrameNum = 30;
    uint32_t specularMaxAccumulatedFrameNum = 30;
    uint32_t diffuseMaxFastAccumulatedFrameNum = 6;
    uint32_t specularMaxFastAccumulatedFrameNum = 6;
    uint32_t historyFixFrameNum = 3;
    uint32_t historyFixBasePixelStride = 14;
    float historyFixEdgeStoppingNormalPower = 8.0f;
    uint32_t spatialVarianceEstimationHistoryThreshold = 3;
    float diffusePrepassBlurRadius = 30.0f;
    float specularPrepassBlurRadius = 50.0f;
    float minHitDistanceWeight = 0.1f;
    float diffusePhiLuminance = 2.0f;
    float specularPhiLuminance = 1.0f;
    float lobeAngleFraction = 0.5f;
    float roughnessFraction = 0.15f;
    float specularVarianceBoost = 0.0f;
    float specularLobeAngleSlack = 0.15f;
    float historyClampingColorBoxSigmaScale = 2.0f;
    uint32_t atrousIterationNum = 5;
    float diffuseMinLuminanceWeight = 0.0f;
    float specularMinLuminanceWeight = 0.0f;
    float depthThreshold = 0.003f;
    float confidenceDrivenRelaxationMultiplier = 0.0f;
    float confidenceDrivenLuminanceEdgeStoppingRelaxation = 0.0f;
    float confidenceDrivenNormalEdgeStoppingRelaxation = 0.0f;
    float luminanceEdgeStoppingRelaxation = 0.5f;
    float normalEdgeStoppingRelaxation = 0.3f;
    float roughnessEdgeStoppingRelaxation = 1.0f;
    CheckerboardMode checkerboardMode = CheckerboardMode::OFF;
    HitDistanceReconstructionMode hitDistanceReconstructionMode = HitDistanceReconstructionMode::OFF;
    bool enableAntiFirefly = false;
    bool enableRoughnessEdgeStopping = true;
    float minMaterialForDiffuse = 4.0f;
    float minMaterialForSpecular = 4.0f;
};

const uint32_t SIGMA_MAX_HISTORY_FRAME_NUM = 7;
const float SIGMA_DEFAULT_ACCUMULATION_TIME = 0.084f;

struct SigmaSettings
{
    float lightDirection[3] = {0.0f, 0.0f, 0.0f};
    float planeDistanceSensitivity = 0.02f;
    uint32_t maxStabilizedFrameNum = 5;
};

const uint32_t REFERENCE_MAX_HISTORY_FRAME_NUM = 4095;
const float REFERENCE_DEFAULT_ACCUMULATION_TIME = 17.0f;
struct ReferenceSettings { uint32_t maxAccumulatedFrameNum = 1020; };

// ---- the nine exported entry points (reference: NRD.h:51-70, Source/Wrapper.cpp:126-303) ------
NRD_API Result NRD_CALL CreateInstance(const InstanceCreationDesc& instanceCreationDesc, Instance*& instance);
NRD_API void NRD_CALL DestroyInstance(Instance& instance);
NRD_API const LibraryDesc& NRD_CALL GetLibraryDesc();
NRD_API const InstanceDesc& NRD_CALL GetInstanceDesc(const Instance& instance);
NRD_API Result NRD_CALL SetCommonSettings(Instance& instance, const CommonSettings& commonSettings);
NRD_API Result NRD_CALL SetDenoiserSettings(Instance& instance, Identifier identifier, const void* denoiserSettings);
// Returned arrays are owned by the instance and overwritten by the next call (NRD.h:64-66).
NRD_API Result NRD_CALL GetComputeDispatches(Instance& instance, const Identifier* identifiers, uint32_t identifiersNum,
                                             const DispatchDesc*& dispatchDescs, uint32_t& dispatchDescsNum);
NRD_API const char* NRD_CALL GetResourceTypeString(ResourceType resourceType);
NRD_API const char* NRD_CALL GetDenoiserString(Denoiser denoiser);
} // namespace nrd

// ---------------------------------------------------------------------------------------------
// Part 2: CUDA executor.  Replaces nrd::Integration::{Initialize,Denoise,Destroy}
// (reference: Integration/NRDIntegration.h:81-131, NRDIntegration.hpp:292-363 pool creation,
// :516-623 Denoise, :625-803 Dispatch).  Plain pointers and sizes only.
//
// One GPU: a context holds the whole frame; pool textures are allocated by the context, IN_*/OUT_* textures are the
// application's own device pointers (nrdCudaSetUserTexture).
// Several GPUs (one process per GPU): the frame is cut into horizontal strips of `stripHeight` rows (a multiple of 16, the
// same on every rank; rank r owns rows [r*stripHeight, min((r+1)*stripHeight, height)) ).  A context then holds only its
// strip of every texture -- pools AND user textures, all carved from one arena that is exported with CUDA IPC -- and the
// owner of a row keeps `haloRows` ghost copies of its boundary rows current in its two neighbours (bulk NVLink stores
// after every pass that writes them); taps that land even further away are loaded directly from the owner's HBM, so the
// result does not depend on the halo size (no recomputation, bit-identical to one GPU).  A device-side flag barrier
// separates the passes.  Kernels address texels in full-frame coordinates in both modes.
// ---------------------------------------------------------------------------------------------
extern "C" {
typedef struct NrdCudaContext NrdCudaContext;

typedef struct NrdCudaContextDesc
{
    uint16_t resourceWidth, resourceHeight;   // full-frame texture size (== CommonSettings::resourceSize)
    uint16_t stripY0, stripY1;                // rows owned by this context; {0, resourceHeight} for one GPU
    uint16_t stripHeight;                     // 0 = one GPU; else the rows reserved per rank (multiple of 16, >= the tallest strip)
    uint16_t haloRows;                        // strip mode: ghost rows kept above/below the strip (rounded up to 16, at least 16, at most stripHeight)
    int32_t device;                          // CUDA device ordinal
} NrdCudaContextDesc;

typedef struct NrdCudaTextureInfo
{
    void* devicePtr;        // address of texel (0, firstRow)
    size_t pitchBytes;
    uint32_t format;        // nrd::Format
    uint16_t width, height; // full (virtual) size of the texture
    uint16_t firstRow, rowsNum; // rows physically present
} NrdCudaTextureInfo;

// Allocates permanentPool[]/transientPool[] of the instance as pitched surfaces on `device`.
NRD_API nrd::Result nrdCudaCreateContext(nrd::Instance* instance, const NrdCudaContextDesc* desc, NrdCudaContext** context);
NRD_API void nrdCudaDestroyContext(NrdCudaContext* context);
// Binds an application texture (IN_* / OUT_*).  Required formats: IN_MV RGBA16_SFLOAT, IN_NORMAL_ROUGHNESS
// R10_G10_B10_A2_UNORM, IN_VIEWZ R32_SFLOAT, IN/OUT_*_RADIANCE_HITDIST RGBA16_SFLOAT, IN_PENUMBRA R16_SFLOAT,
// IN_TRANSLUCENCY RGBA8_UNORM, OUT_SHADOW_TRANSLUCENCY R8_UNORM (SIGMA_SHADOW) / RGBA8_UNORM (SIGMA_SHADOW_TRANSLUCENCY).  `devicePtr` addresses texel (0, firstRow of the context).
// A texture may also be bound in another float format than the one listed (Include/NRDDescs.h lists MINIMUM formats; the listed one is
// what the kernels read): any 16- / 32-bit float format with at least the channels of the listed one (IN_MV may have two), e.g.
// RGBA32_SFLOAT radiance / outputs, R16_SFLOAT viewZ, R16/R32_SFLOAT where R8_UNORM is listed.  The executor keeps a shadow copy in the listed format and converts around the passes (one extra streaming kernel per texture
// and frame).  IN_NORMAL_ROUGHNESS must be the library's normal encoding (LibraryDesc).
NRD_API nrd::Result nrdCudaSetUserTexture(NrdCudaContext* context, uint32_t resourceType, void* devicePtr, size_t pitchBytes, uint32_t format);
// Binds a CUDA array (cudaArray_t / CUarray, level 0 of a mipmapped array, e.g. from
// cudaExternalMemoryGetMappedMipmappedArray + cudaGetMipmappedArrayLevel) as an application texture: the way to reach a Vulkan /
// D3D12 image with optimal tiling.  Formats as for nrdCudaSetUserTexture; texels are the raw bytes of `format`, so the array's
// element size must be BytesPerTexel(format) (R10_G10_B10_A2_UNORM normals: a one-channel 32-bit array).  The array must be 2D (not
// layered, not 3D), created with cudaArraySurfaceLoadStore, and at least resourceWidth x resourceHeight.  The executor keeps a
// pitched shadow in the listed format: nrdCudaDenoise converts every array-bound input into it before the first pass and writes
// every array-bound texture a pass of the frame wrote (outputs, IN_MV on a clear or a TemporalStabilization patch) back after the
// last; nrdCudaExecuteDispatch converts what the dispatch reads before it and what it writes after it.  nrdCudaGetTexture /
// UploadTexture / DownloadTexture act on the shadow.  Binding a type by array or by pointer replaces the previous binding of
// either kind.  Refused: null context or array, or an array smaller than the resource size (INVALID_ARGUMENT); a layered / 3D
// array, no surface load / store, a wrong element size or format, a resource type no supported denoiser uses, a strip-mode
// context (UNSUPPORTED).
NRD_API nrd::Result nrdCudaSetUserTextureArray(NrdCudaContext* context, uint32_t resourceType, void* cudaArray, uint32_t format);
// Looks a texture up exactly like a DispatchDesc resource would be resolved.
NRD_API nrd::Result nrdCudaGetTexture(NrdCudaContext* context, uint32_t resourceType, uint32_t indexInPool, NrdCudaTextureInfo* info);
// Launches the kernel for one DispatchDesc on `stream` (cudaStream_t); the kernel produces the rows the context owns.  In strip
// mode it is followed by the ghost-row refresh of the textures the pass wrote and by one inter-GPU barrier (same stream).
NRD_API nrd::Result nrdCudaExecuteDispatch(NrdCudaContext* context, const nrd::DispatchDesc* dispatch, void* stream);
// GetComputeDispatches + ExecuteDispatch for each, in order.  Returns the number of kernels launched in *launches.
NRD_API nrd::Result nrdCudaDenoise(NrdCudaContext* context, const nrd::Identifier* identifiers, uint32_t identifiersNum, void* stream, uint32_t* launches);
// Synchronous copies between tightly described host buffers and a texture (pool or user) of the context: the rows
// physically present in the context are transferred.  Used to checkpoint / restore the permanent pool and by the tests.
// Strip mode: only the context's own rows are written -- the neighbours' ghost copies of those rows are NOT refreshed (a ghost
// refresh is a collective step of all ranks).  After restoring history textures into connected strip contexts, run one frame with
// AccumulationMode::RESTART or restore every rank's full ghost range through nrdCudaGetTexture / nrdCudaCopyTexture.
NRD_API nrd::Result nrdCudaUploadTexture(NrdCudaContext* context, uint32_t resourceType, uint32_t indexInPool, const void* hostPtr, size_t hostPitchBytes);
NRD_API nrd::Result nrdCudaDownloadTexture(NrdCudaContext* context, uint32_t resourceType, uint32_t indexInPool, void* hostPtr, size_t hostPitchBytes);
// Asynchronous 2D copy (cudaMemcpyDefault: pinned host or device memory) between an application buffer holding the rows
// physically present in the context (`ptr` addresses texel (0, firstRow)) and a texture of the context.
NRD_API nrd::Result nrdCudaCopyTexture(NrdCudaContext* context, uint32_t resourceType, uint32_t indexInPool, void* ptr, size_t pitchBytes, int32_t toContext, void* stream);

// ---- multi-GPU (strip mode) ----
#define NRD_CUDA_IPC_HANDLE_SIZE 64
// The arena of a strip-mode context and its CUDA IPC handle (NRD_CUDA_IPC_HANDLE_SIZE bytes).
NRD_API nrd::Result nrdCudaGetArena(NrdCudaContext* context, void** devicePtr, size_t* bytes);
NRD_API nrd::Result nrdCudaGetIpcHandle(NrdCudaContext* context, void* handleOut);
// Connects the strips: `ipcHandles` = worldSize handles in rank order (entry `rank` is ignored), as gathered with
// torch.distributed / MPI; alternatively `arenas` = worldSize arena pointers that are already addressable from this
// context's device (contexts of one process).  Exactly one of the two is non-null.  `stripStarts` (worldSize + 1 entries:
// first row of every rank's strip, then the frame height) describes a non-uniform, e.g. cost-balanced, partition; every
// strip starts on a multiple of 16, holds at least haloRows rows and at most stripHeight; null = uniform strips.
NRD_API nrd::Result nrdCudaConnectPeers(NrdCudaContext* context, uint32_t rank, uint32_t worldSize, const void* ipcHandles, void* const* arenas,
                                        const uint16_t* stripStarts);

// Enqueues one inter-GPU barrier on `stream` (no-op on one GPU).  nrdCudaDenoise starts with one -- the input strips the
// peers wrote on their streams are complete before the first pass reads them -- and nrdCudaExecuteDispatch ends with one;
// applications that walk the dispatch list themselves call this once per frame before the first dispatch, and AFTER the
// frame's SetCommonSettings: under dynamic resolution with CommonSettings::rectOrigin[1] != 0 connected strips copy the guide
// inputs (IN_VIEWZ, IN_NORMAL_ROUGHNESS, IN_MV and the optional inputs the settings switch on) to the rect origin here, followed
// by a second barrier; a dispatch whose rectOrigin differs from the one seen here returns INVALID_ARGUMENT.
// Memory: every strip-mode context reserves those copies in its arena at creation -- 23 bytes per texel of
// resourceWidth x (stripHeight + 2 x haloRows), rows padded to 256 bytes (about 113 MB per rank for two 3840x2160 strips with
// haloRows 96) -- because the arena is mapped by the peers once.
NRD_API nrd::Result nrdCudaBarrier(NrdCudaContext* context, void* stream);
// Collective: every connected rank calls it with the same table, between two frames -- after the last nrdCudaExecuteDispatch or
// nrdCudaDenoise of a frame and before the next frame's SetCommonSettings / nrdCudaBarrier.  Moves the strip boundaries: `stripStarts`
// follows the rules of nrdCudaConnectPeers (worldSize + 1 entries, the first 0 and the last the frame height; every strip starts on
// a multiple of 16, owns rows, at most stripHeight of them, and every strip but the last holds at least haloRows).  Every texture
// of the context -- histories, transient textures, the IN_* / OUT_* strips -- keeps its contents: its rows move to their new
// owners, so the next frame continues accumulation and computes the same bits as without the move.  Enqueued on `stream` with no
// host synchronisation (three inter-GPU barriers, one copy kernel, one copy back); the stripY0 / stripY1 of the context change with
// it.  Afterwards the application writes the next frame's IN_* rows, and reads OUT_* rows, through nrdCudaGetTexture /
// nrdCudaCopyTexture with the new firstRow / rowsNum; a dispatch before the next frame start returns FAILURE.
// The library does not choose cuts: see strips.StripDenoiser for a policy.  A larger stripHeight at creation is what makes uneven
// cuts possible, and the arena grows in proportion to it.  Memory: a scratch buffer the size of the arena, allocated and freed
// on `stream` (cudaMallocAsync), exists only while the call runs.
// INVALID_ARGUMENT: null context or table, or a table that breaks the rules -- refused before anything is enqueued, alike on every
// rank.  UNSUPPORTED: a one-GPU context, or a strip context that is not connected.  FAILURE: an earlier barrier of the context
// timed out.  A connected world of one accepts the identity table only, and does nothing.
NRD_API nrd::Result nrdCudaRepartition(NrdCudaContext* context, const uint16_t* stripStarts, void* stream);
// cudaStreamSynchronize + check that no inter-GPU barrier timed out (a peer that died or fell out of step).
NRD_API nrd::Result nrdCudaSynchronize(NrdCudaContext* context, void* stream);

// Last CUDA error string seen by the executor ("" if none).
// Profiling aid (multi-GPU balance): with timing on, every dispatch of nrdCudaDenoise / nrdCudaExecuteDispatch is bracketed by CUDA
// events on its stream -- kernelMs[i] = the pass kernel alone, exchangeMs[i] = its ghost-row push + inter-GPU barrier (i.e. the
// NVLink copy plus the wait for the slowest neighbour).  nrdCudaGetTiming synchronises the events recorded since the last call
// (at most 64 dispatches are kept) and returns how many there were.  Frames of connected strips with rectOrigin[1] != 0 add two
// slots: the first of the frame is the copy of the guide inputs to the rect origin (exchangeMs = the barrier after it), and the
// slot right after REBLUR temporal stabilization with isBaseColorMetalnessAvailable is the copy of IN_MV back to the
// application's strip (exchangeMs = 0).  Clear dispatches are not timed.
NRD_API nrd::Result nrdCudaSetTiming(NrdCudaContext* context, int32_t enable);
NRD_API nrd::Result nrdCudaGetTiming(NrdCudaContext* context, float* kernelMs, float* exchangeMs, uint32_t capacity, uint32_t* count);
NRD_API const char* nrdCudaGetLastError(NrdCudaContext* context);
// Total kernels launched by this library in the process (for bench.py's gpu_launches).
NRD_API uint64_t nrdCudaGetLaunchCount();
}
