"""Host-side mirror of the NRD interface (reference: Include/NRD.h, NRDDescs.h, NRDSettings.h) over the C-ABI of
libnrd_b200.so (include/nrd_b200.h).  Same names, same argument meaning, same Result codes as the reference so that
code written against `nrd::` reads the same here:

    inst = nrd.Instance([(0, nrd.Denoiser.REBLUR_DIFFUSE_SPECULAR)])
    inst.set_common_settings(cs); inst.set_denoiser_settings(0, nrd.ReblurSettings())
    dispatches = inst.get_compute_dispatches([0])

The CUDA executor (nrdCuda*) replaces the reference's NRI integration layer.  Nothing here computes anything: the
library is the product, this file is plumbing.  It fails loudly if the native library is missing.
"""
import ctypes as C
import enum
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.environ.get("NRD_B200_LIB") or os.path.join(_HERE, "libnrd_b200.so")  # the override is for A/B kernel builds


def _load():
    if not os.path.exists(_LIB_PATH):
        raise ImportError("libnrd_b200.so is not built; run `python -m raytracingdenoiser_b200.build` (there is no fallback path)")
    return C.CDLL(_LIB_PATH)


_lib = _load()


class Result(enum.IntEnum):
    SUCCESS = 0
    FAILURE = 1
    INVALID_ARGUMENT = 2
    UNSUPPORTED = 3
    NON_UNIQUE_IDENTIFIER = 4


_RESOURCE_TYPES = """IN_MV IN_NORMAL_ROUGHNESS IN_VIEWZ IN_DIFF_CONFIDENCE IN_SPEC_CONFIDENCE IN_DISOCCLUSION_THRESHOLD_MIX
IN_BASECOLOR_METALNESS IN_DIFF_RADIANCE_HITDIST IN_SPEC_RADIANCE_HITDIST IN_DIFF_HITDIST IN_SPEC_HITDIST IN_DIFF_DIRECTION_HITDIST
IN_DIFF_SH0 IN_DIFF_SH1 IN_SPEC_SH0 IN_SPEC_SH1 IN_PENUMBRA IN_TRANSLUCENCY IN_SIGNAL OUT_DIFF_RADIANCE_HITDIST OUT_SPEC_RADIANCE_HITDIST
OUT_DIFF_SH0 OUT_DIFF_SH1 OUT_SPEC_SH0 OUT_SPEC_SH1 OUT_DIFF_HITDIST OUT_SPEC_HITDIST OUT_DIFF_DIRECTION_HITDIST OUT_SHADOW_TRANSLUCENCY
OUT_SIGNAL OUT_VALIDATION TRANSIENT_POOL PERMANENT_POOL""".split()
ResourceType = enum.IntEnum("ResourceType", {n: i for i, n in enumerate(_RESOURCE_TYPES)})

_DENOISERS = """REBLUR_DIFFUSE REBLUR_DIFFUSE_OCCLUSION REBLUR_DIFFUSE_SH REBLUR_SPECULAR REBLUR_SPECULAR_OCCLUSION REBLUR_SPECULAR_SH
REBLUR_DIFFUSE_SPECULAR REBLUR_DIFFUSE_SPECULAR_OCCLUSION REBLUR_DIFFUSE_SPECULAR_SH REBLUR_DIFFUSE_DIRECTIONAL_OCCLUSION RELAX_DIFFUSE
RELAX_DIFFUSE_SH RELAX_SPECULAR RELAX_SPECULAR_SH RELAX_DIFFUSE_SPECULAR RELAX_DIFFUSE_SPECULAR_SH SIGMA_SHADOW SIGMA_SHADOW_TRANSLUCENCY
REFERENCE""".split()
Denoiser = enum.IntEnum("Denoiser", {n: i for i, n in enumerate(_DENOISERS)})

_FORMATS = """R8_UNORM R8_SNORM R8_UINT R8_SINT RG8_UNORM RG8_SNORM RG8_UINT RG8_SINT RGBA8_UNORM RGBA8_SNORM RGBA8_UINT RGBA8_SINT RGBA8_SRGB
R16_UNORM R16_SNORM R16_UINT R16_SINT R16_SFLOAT RG16_UNORM RG16_SNORM RG16_UINT RG16_SINT RG16_SFLOAT RGBA16_UNORM RGBA16_SNORM RGBA16_UINT
RGBA16_SINT RGBA16_SFLOAT R32_UINT R32_SINT R32_SFLOAT RG32_UINT RG32_SINT RG32_SFLOAT RGB32_UINT RGB32_SINT RGB32_SFLOAT RGBA32_UINT RGBA32_SINT
RGBA32_SFLOAT R10_G10_B10_A2_UNORM R10_G10_B10_A2_UINT R11_G11_B10_UFLOAT R9_G9_B9_E5_UFLOAT""".split()
Format = enum.IntEnum("Format", {n: i for i, n in enumerate(_FORMATS)})
FORMAT_BYTES = {Format.R8_UNORM: 1, Format.R8_UINT: 1, Format.RG8_UNORM: 2, Format.RGBA8_UNORM: 4, Format.R16_UNORM: 2, Format.R16_UINT: 2,
                Format.R16_SFLOAT: 2, Format.RGBA16_SFLOAT: 8, Format.R32_UINT: 4, Format.R32_SFLOAT: 4, Format.R10_G10_B10_A2_UNORM: 4}


class DescriptorType(enum.IntEnum):
    TEXTURE = 0
    STORAGE_TEXTURE = 1


class CheckerboardMode(enum.IntEnum):
    OFF = 0
    BLACK = 1
    WHITE = 2


class AccumulationMode(enum.IntEnum):
    CONTINUE = 0
    RESTART = 1
    CLEAR_AND_RESTART = 2


class HitDistanceReconstructionMode(enum.IntEnum):
    OFF = 0
    AREA_3X3 = 1
    AREA_5X5 = 2


def _struct(name, fields, defaults=None):
    """ctypes Structure whose constructor applies the reference's default member initialisers."""
    defaults = defaults or {}

    def __init__(self, **kw):
        C.Structure.__init__(self)
        for k, v in defaults.items():
            _assign(self, k, v)
        for k, v in kw.items():
            _assign(self, k, v)

    return type(name, (C.Structure,), {"_fields_": fields, "__init__": __init__})


def _assign(obj, key, value):
    cur = getattr(obj, key)
    if isinstance(cur, C.Array):
        for i, v in enumerate(value):
            cur[i] = v
    else:
        setattr(obj, key, value)


f32, u8, u16, u32, b8 = C.c_float, C.c_uint8, C.c_uint16, C.c_uint32, C.c_bool

AllocationCallbacks = _struct("AllocationCallbacks", [("Allocate", C.c_void_p), ("Reallocate", C.c_void_p), ("Free", C.c_void_p), ("userArg", C.c_void_p)])
SPIRVBindingOffsets = _struct("SPIRVBindingOffsets", [("samplerOffset", u32), ("textureOffset", u32), ("constantBufferOffset", u32), ("storageTextureAndBufferOffset", u32)])
LibraryDesc = _struct("LibraryDesc", [("spirvBindingOffsets", SPIRVBindingOffsets), ("supportedDenoisers", C.POINTER(u32)), ("supportedDenoisersNum", u32),
                                      ("versionMajor", u8), ("versionMinor", u8), ("versionBuild", u8), ("normalEncoding", u8), ("roughnessEncoding", u8)])
DenoiserDesc = _struct("DenoiserDesc", [("identifier", u32), ("denoiser", u32)])
InstanceCreationDesc = _struct("InstanceCreationDesc", [("allocationCallbacks", AllocationCallbacks), ("denoisers", C.POINTER(DenoiserDesc)), ("denoisersNum", u32)])
TextureDesc = _struct("TextureDesc", [("format", u32), ("downsampleFactor", u16)])
ResourceDesc = _struct("ResourceDesc", [("descriptorType", u32), ("type", u32), ("indexInPool", u16)])
ResourceRangeDesc = _struct("ResourceRangeDesc", [("descriptorType", u32), ("baseRegisterIndex", u32), ("descriptorsNum", u32)])
ComputeShaderDesc = _struct("ComputeShaderDesc", [("bytecode", C.c_void_p), ("size", C.c_uint64)])
PipelineDesc = _struct("PipelineDesc", [("computeShaderDXBC", ComputeShaderDesc), ("computeShaderDXIL", ComputeShaderDesc), ("computeShaderSPIRV", ComputeShaderDesc),
                                        ("shaderFileName", C.c_char_p), ("shaderEntryPointName", C.c_char_p), ("resourceRanges", C.POINTER(ResourceRangeDesc)),
                                        ("resourceRangesNum", u32), ("hasConstantData", b8)])
DescriptorPoolDesc = _struct("DescriptorPoolDesc", [("setsMaxNum", u32), ("constantBuffersMaxNum", u32), ("samplersMaxNum", u32), ("texturesMaxNum", u32), ("storageTexturesMaxNum", u32)])
InstanceDesc = _struct("InstanceDesc", [("constantBufferMaxDataSize", u32), ("constantBufferSpaceIndex", u32), ("constantBufferRegisterIndex", u32),
                                        ("samplers", C.POINTER(u32)), ("samplersNum", u32), ("samplersSpaceIndex", u32), ("samplersBaseRegisterIndex", u32),
                                        ("pipelines", C.POINTER(PipelineDesc)), ("pipelinesNum", u32), ("resourcesSpaceIndex", u32),
                                        ("permanentPool", C.POINTER(TextureDesc)), ("permanentPoolSize", u32), ("transientPool", C.POINTER(TextureDesc)),
                                        ("transientPoolSize", u32), ("descriptorPoolDesc", DescriptorPoolDesc)])
DispatchDesc = _struct("DispatchDesc", [("name", C.c_char_p), ("identifier", u32), ("resources", C.POINTER(ResourceDesc)), ("resourcesNum", u32),
                                        ("constantBufferData", C.POINTER(u8)), ("constantBufferDataSize", u32), ("constantBufferDataMatchesPreviousDispatch", b8),
                                        ("pipelineIndex", u16), ("gridWidth", u16), ("gridHeight", u16)])

_IDENTITY = [1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1]
CommonSettings = _struct("CommonSettings", [
    ("viewToClipMatrix", f32 * 16), ("viewToClipMatrixPrev", f32 * 16), ("worldToViewMatrix", f32 * 16), ("worldToViewMatrixPrev", f32 * 16),
    ("worldPrevToWorldMatrix", f32 * 16), ("motionVectorScale", f32 * 3), ("cameraJitter", f32 * 2), ("cameraJitterPrev", f32 * 2),
    ("resourceSize", u16 * 2), ("resourceSizePrev", u16 * 2), ("rectSize", u16 * 2), ("rectSizePrev", u16 * 2),
    ("viewZScale", f32), ("timeDeltaBetweenFrames", f32), ("denoisingRange", f32), ("disocclusionThreshold", f32), ("disocclusionThresholdAlternate", f32),
    ("cameraAttachedReflectionMaterialID", f32), ("strandMaterialID", f32), ("strandThickness", f32), ("splitScreen", f32),
    ("printfAt", u16 * 2), ("debug", f32), ("rectOrigin", u32 * 2), ("frameIndex", u32), ("accumulationMode", u8),
    ("isMotionVectorInWorldSpace", b8), ("isHistoryConfidenceAvailable", b8), ("isDisocclusionThresholdMixAvailable", b8),
    ("isBaseColorMetalnessAvailable", b8), ("enableValidation", b8)],
    dict(worldPrevToWorldMatrix=_IDENTITY, motionVectorScale=[1.0, 1.0, 0.0], viewZScale=1.0, denoisingRange=500000.0, disocclusionThreshold=0.01,
         disocclusionThresholdAlternate=0.05, cameraAttachedReflectionMaterialID=999.0, strandMaterialID=999.0, strandThickness=80e-6, printfAt=[9999, 9999]))

HitDistanceParameters = _struct("HitDistanceParameters", [("A", f32), ("B", f32), ("C", f32), ("D", f32)], dict(A=3.0, B=0.1, C=20.0, D=-25.0))
ReblurAntilagSettings = _struct("ReblurAntilagSettings", [("luminanceSigmaScale", f32), ("luminanceSensitivity", f32)], dict(luminanceSigmaScale=4.0, luminanceSensitivity=3.0))
ReblurSettings = _struct("ReblurSettings", [
    ("hitDistanceParameters", HitDistanceParameters), ("antilagSettings", ReblurAntilagSettings), ("maxAccumulatedFrameNum", u32),
    ("maxFastAccumulatedFrameNum", u32), ("maxStabilizedFrameNum", u32), ("maxStabilizedFrameNumForHitDistance", u32), ("historyFixFrameNum", u32),
    ("historyFixBasePixelStride", u32), ("diffusePrepassBlurRadius", f32), ("specularPrepassBlurRadius", f32), ("minHitDistanceWeight", f32),
    ("minBlurRadius", f32), ("maxBlurRadius", f32), ("lobeAngleFraction", f32), ("roughnessFraction", f32), ("responsiveAccumulationRoughnessThreshold", f32),
    ("planeDistanceSensitivity", f32), ("specularProbabilityThresholdsForMvModification", f32 * 2), ("fireflySuppressorMinRelativeScale", f32),
    ("checkerboardMode", u8), ("hitDistanceReconstructionMode", u8), ("enableAntiFirefly", b8), ("enablePerformanceMode", b8),
    ("minMaterialForDiffuse", f32), ("minMaterialForSpecular", f32), ("usePrepassOnlyForSpecularMotionEstimation", b8)],
    dict(hitDistanceParameters=HitDistanceParameters(), antilagSettings=ReblurAntilagSettings(), maxAccumulatedFrameNum=30, maxFastAccumulatedFrameNum=6,
         maxStabilizedFrameNum=63, maxStabilizedFrameNumForHitDistance=63, historyFixFrameNum=3, historyFixBasePixelStride=14, diffusePrepassBlurRadius=30.0,
         specularPrepassBlurRadius=50.0, minHitDistanceWeight=0.1, minBlurRadius=1.0, maxBlurRadius=30.0, lobeAngleFraction=0.15, roughnessFraction=0.15,
         planeDistanceSensitivity=0.02, specularProbabilityThresholdsForMvModification=[0.5, 0.9], fireflySuppressorMinRelativeScale=2.0,
         minMaterialForDiffuse=4.0, minMaterialForSpecular=4.0))

RelaxAntilagSettings = _struct("RelaxAntilagSettings", [("accelerationAmount", f32), ("spatialSigmaScale", f32), ("temporalSigmaScale", f32), ("resetAmount", f32)],
                               dict(accelerationAmount=0.3, spatialSigmaScale=4.5, temporalSigmaScale=0.5, resetAmount=0.5))
RelaxSettings = _struct("RelaxSettings", [
    ("antilagSettings", RelaxAntilagSettings), ("diffuseMaxAccumulatedFrameNum", u32), ("specularMaxAccumulatedFrameNum", u32),
    ("diffuseMaxFastAccumulatedFrameNum", u32), ("specularMaxFastAccumulatedFrameNum", u32), ("historyFixFrameNum", u32), ("historyFixBasePixelStride", u32),
    ("historyFixEdgeStoppingNormalPower", f32), ("spatialVarianceEstimationHistoryThreshold", u32), ("diffusePrepassBlurRadius", f32),
    ("specularPrepassBlurRadius", f32), ("minHitDistanceWeight", f32), ("diffusePhiLuminance", f32), ("specularPhiLuminance", f32), ("lobeAngleFraction", f32),
    ("roughnessFraction", f32), ("specularVarianceBoost", f32), ("specularLobeAngleSlack", f32), ("historyClampingColorBoxSigmaScale", f32),
    ("atrousIterationNum", u32), ("diffuseMinLuminanceWeight", f32), ("specularMinLuminanceWeight", f32), ("depthThreshold", f32),
    ("confidenceDrivenRelaxationMultiplier", f32), ("confidenceDrivenLuminanceEdgeStoppingRelaxation", f32), ("confidenceDrivenNormalEdgeStoppingRelaxation", f32),
    ("luminanceEdgeStoppingRelaxation", f32), ("normalEdgeStoppingRelaxation", f32), ("roughnessEdgeStoppingRelaxation", f32), ("checkerboardMode", u8),
    ("hitDistanceReconstructionMode", u8), ("enableAntiFirefly", b8), ("enableRoughnessEdgeStopping", b8), ("minMaterialForDiffuse", f32),
    ("minMaterialForSpecular", f32)],
    dict(antilagSettings=RelaxAntilagSettings(), diffuseMaxAccumulatedFrameNum=30, specularMaxAccumulatedFrameNum=30, diffuseMaxFastAccumulatedFrameNum=6,
         specularMaxFastAccumulatedFrameNum=6, historyFixFrameNum=3, historyFixBasePixelStride=14, historyFixEdgeStoppingNormalPower=8.0,
         spatialVarianceEstimationHistoryThreshold=3, diffusePrepassBlurRadius=30.0, specularPrepassBlurRadius=50.0, minHitDistanceWeight=0.1,
         diffusePhiLuminance=2.0, specularPhiLuminance=1.0, lobeAngleFraction=0.5, roughnessFraction=0.15, specularLobeAngleSlack=0.15,
         historyClampingColorBoxSigmaScale=2.0, atrousIterationNum=5, depthThreshold=0.003, luminanceEdgeStoppingRelaxation=0.5,
         normalEdgeStoppingRelaxation=0.3, roughnessEdgeStoppingRelaxation=1.0, enableRoughnessEdgeStopping=True, minMaterialForDiffuse=4.0,
         minMaterialForSpecular=4.0))

SigmaSettings = _struct("SigmaSettings", [("lightDirection", f32 * 3), ("planeDistanceSensitivity", f32), ("maxStabilizedFrameNum", u32)],
                        dict(planeDistanceSensitivity=0.02, maxStabilizedFrameNum=5))

ReferenceSettings = _struct("ReferenceSettings", [("maxAccumulatedFrameNum", u32)], dict(maxAccumulatedFrameNum=1020))

NrdCudaContextDesc = _struct("NrdCudaContextDesc", [("resourceWidth", u16), ("resourceHeight", u16), ("stripY0", u16), ("stripY1", u16), ("stripHeight", u16), ("haloRows", u16), ("device", C.c_int32)])
NrdCudaTextureInfo = _struct("NrdCudaTextureInfo", [("devicePtr", C.c_void_p), ("pitchBytes", C.c_size_t), ("format", u32), ("width", u16), ("height", u16),
                                                    ("firstRow", u16), ("rowsNum", u16)])

# ---- prototypes ---------------------------------------------------------------------------------------
def bind_nrd_api(lib):
    """Declares the prototypes of the nine NRD entry points (Include/NRD.h:51-70) on `lib`.  Used for libnrd_b200.so and, in
    tests/test_reference_scheduler.py, for the reference's own host library built by oracle/Makefile.ref."""
    lib.CreateInstance.argtypes = [C.POINTER(InstanceCreationDesc), C.POINTER(C.c_void_p)]
    lib.CreateInstance.restype = u32
    lib.DestroyInstance.argtypes = [C.c_void_p]
    lib.DestroyInstance.restype = None
    lib.GetLibraryDesc.argtypes = []
    lib.GetLibraryDesc.restype = C.POINTER(LibraryDesc)
    lib.GetInstanceDesc.argtypes = [C.c_void_p]
    lib.GetInstanceDesc.restype = C.POINTER(InstanceDesc)
    lib.SetCommonSettings.argtypes = [C.c_void_p, C.POINTER(CommonSettings)]
    lib.SetCommonSettings.restype = u32
    lib.SetDenoiserSettings.argtypes = [C.c_void_p, u32, C.c_void_p]
    lib.SetDenoiserSettings.restype = u32
    lib.GetComputeDispatches.argtypes = [C.c_void_p, C.POINTER(u32), u32, C.POINTER(C.POINTER(DispatchDesc)), C.POINTER(u32)]
    lib.GetComputeDispatches.restype = u32
    lib.GetResourceTypeString.argtypes = [u32]
    lib.GetResourceTypeString.restype = C.c_char_p
    lib.GetDenoiserString.argtypes = [u32]
    lib.GetDenoiserString.restype = C.c_char_p
    return lib


bind_nrd_api(_lib)
_lib.nrdCudaCreateContext.argtypes = [C.c_void_p, C.POINTER(NrdCudaContextDesc), C.POINTER(C.c_void_p)]
_lib.nrdCudaCreateContext.restype = u32
_lib.nrdCudaDestroyContext.argtypes = [C.c_void_p]
_lib.nrdCudaDestroyContext.restype = None
_lib.nrdCudaSetUserTexture.argtypes = [C.c_void_p, u32, C.c_void_p, C.c_size_t, u32]
_lib.nrdCudaSetUserTexture.restype = u32
_lib.nrdCudaSetUserTextureArray.argtypes = [C.c_void_p, u32, C.c_void_p, u32]
_lib.nrdCudaSetUserTextureArray.restype = u32
_lib.nrdCudaGetTexture.argtypes = [C.c_void_p, u32, u32, C.POINTER(NrdCudaTextureInfo)]
_lib.nrdCudaGetTexture.restype = u32
_lib.nrdCudaExecuteDispatch.argtypes = [C.c_void_p, C.POINTER(DispatchDesc), C.c_void_p]
_lib.nrdCudaExecuteDispatch.restype = u32
_lib.nrdCudaDenoise.argtypes = [C.c_void_p, C.POINTER(u32), u32, C.c_void_p, C.POINTER(u32)]
_lib.nrdCudaDenoise.restype = u32
_lib.nrdCudaUploadTexture.argtypes = [C.c_void_p, u32, u32, C.c_void_p, C.c_size_t]
_lib.nrdCudaUploadTexture.restype = u32
_lib.nrdCudaDownloadTexture.argtypes = [C.c_void_p, u32, u32, C.c_void_p, C.c_size_t]
_lib.nrdCudaDownloadTexture.restype = u32
_lib.nrdCudaGetLastError.argtypes = [C.c_void_p]
_lib.nrdCudaGetLastError.restype = C.c_char_p
_lib.nrdCudaGetLaunchCount.argtypes = []
_lib.nrdCudaGetLaunchCount.restype = C.c_uint64
_lib.nrdCudaCopyTexture.argtypes = [C.c_void_p, u32, u32, C.c_void_p, C.c_size_t, C.c_int32, C.c_void_p]
_lib.nrdCudaCopyTexture.restype = u32
_lib.nrdCudaGetArena.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_size_t)]
_lib.nrdCudaGetArena.restype = u32
_lib.nrdCudaGetIpcHandle.argtypes = [C.c_void_p, C.c_void_p]
_lib.nrdCudaGetIpcHandle.restype = u32
_lib.nrdCudaConnectPeers.argtypes = [C.c_void_p, u32, u32, C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(u16)]
_lib.nrdCudaConnectPeers.restype = u32
_lib.nrdCudaBarrier.argtypes = [C.c_void_p, C.c_void_p]
_lib.nrdCudaBarrier.restype = u32
_lib.nrdCudaRepartition.argtypes = [C.c_void_p, C.POINTER(u16), C.c_void_p]
_lib.nrdCudaRepartition.restype = u32
_lib.nrdCudaSynchronize.argtypes = [C.c_void_p, C.c_void_p]
_lib.nrdCudaSynchronize.restype = u32
_lib.nrdCudaSetTiming.argtypes = [C.c_void_p, C.c_int32]
_lib.nrdCudaSetTiming.restype = u32
_lib.nrdCudaGetTiming.argtypes = [C.c_void_p, C.POINTER(C.c_float), C.POINTER(C.c_float), C.c_uint32, C.POINTER(C.c_uint32)]
_lib.nrdCudaGetTiming.restype = u32
IPC_HANDLE_SIZE = 64

EXPORTED_SYMBOLS = ["CreateInstance", "DestroyInstance", "GetLibraryDesc", "GetInstanceDesc", "SetCommonSettings", "SetDenoiserSettings",
                    "GetComputeDispatches", "GetResourceTypeString", "GetDenoiserString", "nrdCudaCreateContext", "nrdCudaDestroyContext",
                    "nrdCudaSetUserTexture", "nrdCudaSetUserTextureArray", "nrdCudaGetTexture", "nrdCudaExecuteDispatch", "nrdCudaDenoise", "nrdCudaUploadTexture", "nrdCudaDownloadTexture", "nrdCudaGetLastError", "nrdCudaGetLaunchCount",
                    "nrdCudaCopyTexture", "nrdCudaGetArena", "nrdCudaGetIpcHandle", "nrdCudaConnectPeers", "nrdCudaBarrier", "nrdCudaSynchronize", "nrdCudaSetTiming", "nrdCudaGetTiming"]


class NrdError(RuntimeError):
    def __init__(self, what, result):
        RuntimeError.__init__(self, "%s -> Result::%s" % (what, Result(result).name))
        self.result = Result(result)


def library_path():
    return _LIB_PATH


def get_library_desc():
    d = _lib.GetLibraryDesc().contents
    return {"versionMajor": d.versionMajor, "versionMinor": d.versionMinor, "versionBuild": d.versionBuild, "normalEncoding": d.normalEncoding,
            "roughnessEncoding": d.roughnessEncoding, "supportedDenoisers": [Denoiser(d.supportedDenoisers[i]) for i in range(d.supportedDenoisersNum)],
            "spirvBindingOffsets": (d.spirvBindingOffsets.samplerOffset, d.spirvBindingOffsets.textureOffset, d.spirvBindingOffsets.constantBufferOffset,
                                    d.spirvBindingOffsets.storageTextureAndBufferOffset)}


def get_resource_type_string(t):
    s = _lib.GetResourceTypeString(int(t))
    return s.decode() if s else None


def get_denoiser_string(d):
    s = _lib.GetDenoiserString(int(d))
    return s.decode() if s else None


class Dispatch(object):
    """One DispatchDesc copied out of instance-owned memory (it is overwritten by the next GetComputeDispatches)."""

    def __init__(self, raw, pipelines):
        self.name = raw.name.decode()
        self.identifier = raw.identifier
        self.resources = [(DescriptorType(raw.resources[i].descriptorType), ResourceType(raw.resources[i].type), raw.resources[i].indexInPool)
                          for i in range(raw.resourcesNum)]
        self.constants = bytes(bytearray(raw.constantBufferData[:raw.constantBufferDataSize])) if raw.constantBufferDataSize else b""
        self.constantsMatchPrevious = bool(raw.constantBufferDataMatchesPreviousDispatch)
        self.pipelineIndex = raw.pipelineIndex
        self.shaderFileName = pipelines[raw.pipelineIndex]["shaderFileName"]
        self.gridWidth = raw.gridWidth
        self.gridHeight = raw.gridHeight

    def __repr__(self):
        return "Dispatch(%r, %s, grid=%dx%d, %d resources)" % (self.name, self.shaderFileName, self.gridWidth, self.gridHeight, len(self.resources))


class Instance(object):
    """nrd::Instance (reference: CreateInstance / DestroyInstance, Source/Wrapper.cpp:246-289)."""

    def __init__(self, denoisers, lib=None):
        self._lib = lib or _lib   # `lib`: another library exporting the NRD API (the reference build, tests only)
        arr = (DenoiserDesc * len(denoisers))()
        for i, (identifier, denoiser) in enumerate(denoisers):
            arr[i].identifier = identifier
            arr[i].denoiser = int(denoiser)
        desc = InstanceCreationDesc()
        desc.denoisers = arr
        desc.denoisersNum = len(denoisers)
        self._handle = C.c_void_p()
        r = self._lib.CreateInstance(C.byref(desc), C.byref(self._handle))
        if r != Result.SUCCESS:
            self._handle = None
            raise NrdError("CreateInstance", r)
        self.denoisers = list(denoisers)

    def destroy(self):
        if self._handle:
            self._lib.DestroyInstance(self._handle)
            self._handle = None

    def __del__(self):
        try:
            self.destroy()
        except Exception:
            pass

    @property
    def handle(self):
        return self._handle

    def get_instance_desc(self):
        d = self._lib.GetInstanceDesc(self._handle).contents
        pipelines = []
        for i in range(d.pipelinesNum):
            p = d.pipelines[i]
            pipelines.append({"shaderFileName": p.shaderFileName.decode(), "shaderEntryPointName": p.shaderEntryPointName.decode(),
                              "hasConstantData": bool(p.hasConstantData), "bytecodeSizes": (p.computeShaderDXBC.size, p.computeShaderDXIL.size, p.computeShaderSPIRV.size),
                              "resourceRanges": [(DescriptorType(p.resourceRanges[j].descriptorType), p.resourceRanges[j].descriptorsNum) for j in range(p.resourceRangesNum)]})
        return {"constantBufferMaxDataSize": d.constantBufferMaxDataSize, "samplersNum": d.samplersNum, "pipelines": pipelines,
                "permanentPool": [(Format(d.permanentPool[i].format), d.permanentPool[i].downsampleFactor) for i in range(d.permanentPoolSize)],
                "transientPool": [(Format(d.transientPool[i].format), d.transientPool[i].downsampleFactor) for i in range(d.transientPoolSize)],
                "descriptorPoolDesc": {k: getattr(d.descriptorPoolDesc, k) for k, _ in DescriptorPoolDesc._fields_}}

    def set_common_settings(self, common_settings, check=True):
        r = Result(self._lib.SetCommonSettings(self._handle, C.byref(common_settings)))
        if check and r != Result.SUCCESS:
            raise NrdError("SetCommonSettings", r)
        return r

    def set_denoiser_settings(self, identifier, settings, check=True):
        r = Result(self._lib.SetDenoiserSettings(self._handle, identifier, C.byref(settings)))
        if check and r != Result.SUCCESS:
            raise NrdError("SetDenoiserSettings", r)
        return r

    def get_compute_dispatches_raw(self, identifiers):
        ids = (u32 * max(len(identifiers), 1))(*identifiers)
        out = C.POINTER(DispatchDesc)()
        num = u32(0)
        r = Result(self._lib.GetComputeDispatches(self._handle, ids if identifiers else None, len(identifiers), C.byref(out), C.byref(num)))
        return r, out, num.value

    def get_compute_dispatches(self, identifiers, check=True):
        r, out, n = self.get_compute_dispatches_raw(identifiers)
        if check and r != Result.SUCCESS:
            raise NrdError("GetComputeDispatches", r)
        pipelines = self.get_instance_desc()["pipelines"] if n else []
        return [Dispatch(out[i], pipelines) for i in range(n)]


class CudaContext(object):
    """CUDA executor for one Instance (replaces nrd::Integration).  Textures are plain device pointers + pitch, or CUDA arrays."""

    def __init__(self, instance, width, height, device=0, strip=None, strip_height=0, halo_rows=0):
        """strip=(y0, y1), strip_height=S, halo_rows=H: strip-mode context of a multi-GPU run (see include/nrd_b200.h)."""
        desc = NrdCudaContextDesc()
        desc.resourceWidth, desc.resourceHeight = width, height
        desc.stripY0, desc.stripY1 = strip if strip else (0, height)
        desc.stripHeight = strip_height
        desc.haloRows = halo_rows
        desc.device = device
        self.strip = (desc.stripY0, desc.stripY1)
        self.strip_height = strip_height
        self.world_size = None  # set by connect_peers
        self.instance = instance
        self.width, self.height = width, height
        self._ctx = C.c_void_p()
        r = _lib.nrdCudaCreateContext(instance.handle, C.byref(desc), C.byref(self._ctx))
        if r != Result.SUCCESS:
            self._ctx = None
            raise NrdError("nrdCudaCreateContext (is a CUDA device visible?)", r)

    def destroy(self):
        if self._ctx:
            _lib.nrdCudaDestroyContext(self._ctx)
            self._ctx = None

    def __del__(self):
        try:
            self.destroy()
        except Exception:
            pass

    def _check(self, what, r):
        if r != Result.SUCCESS:
            msg = _lib.nrdCudaGetLastError(self._ctx)
            raise NrdError("%s [%s]" % (what, msg.decode() if msg else ""), r)

    def set_user_texture(self, resource_type, device_ptr, pitch_bytes, fmt):
        self._check("nrdCudaSetUserTexture(%s)" % ResourceType(resource_type).name,
                    _lib.nrdCudaSetUserTexture(self._ctx, int(resource_type), C.c_void_p(device_ptr), pitch_bytes, int(fmt)))

    def set_user_texture_array(self, resource_type, array_handle, fmt):
        """array_handle: a cudaArray_t / CUarray as an int (level 0 of a mipmapped array, e.g. an imported Vulkan / D3D12 image)
        created with surface load / store; the executor converts it to and from a shadow in the kernels' format around the passes."""
        self._check("nrdCudaSetUserTextureArray(%s)" % ResourceType(resource_type).name,
                    _lib.nrdCudaSetUserTextureArray(self._ctx, int(resource_type), C.c_void_p(array_handle), int(fmt)))

    def get_texture(self, resource_type, index_in_pool=0):
        info = NrdCudaTextureInfo()
        self._check("nrdCudaGetTexture", _lib.nrdCudaGetTexture(self._ctx, int(resource_type), index_in_pool, C.byref(info)))
        return info

    def upload(self, resource_type, index_in_pool, array):
        """array: C-contiguous numpy array whose rows are the texture rows (row stride = array.strides[0])."""
        self._check("nrdCudaUploadTexture", _lib.nrdCudaUploadTexture(self._ctx, int(resource_type), index_in_pool, array.ctypes.data, array.strides[0]))

    def download(self, resource_type, index_in_pool, array):
        self._check("nrdCudaDownloadTexture", _lib.nrdCudaDownloadTexture(self._ctx, int(resource_type), index_in_pool, array.ctypes.data, array.strides[0]))

    def copy(self, resource_type, index_in_pool, ptr, pitch_bytes, to_context, stream=0):
        """Async 2D copy of the rows held by the context between a device / pinned-host buffer and a texture."""
        self._check("nrdCudaCopyTexture", _lib.nrdCudaCopyTexture(self._ctx, int(resource_type), index_in_pool, C.c_void_p(ptr), pitch_bytes, 1 if to_context else 0,
                                                                   C.c_void_p(stream)))

    def arena(self):
        ptr, size = C.c_void_p(), C.c_size_t()
        self._check("nrdCudaGetArena", _lib.nrdCudaGetArena(self._ctx, C.byref(ptr), C.byref(size)))
        return ptr.value, size.value

    def ipc_handle(self):
        buf = C.create_string_buffer(IPC_HANDLE_SIZE)
        self._check("nrdCudaGetIpcHandle", _lib.nrdCudaGetIpcHandle(self._ctx, buf))
        return buf.raw

    def connect_peers(self, rank, world_size, ipc_handles=None, arenas=None, strip_starts=None):
        """ipc_handles: list of world_size 64-byte handles (other processes); arenas: list of arena pointers (same process);
        strip_starts: world_size + 1 row indices of a non-uniform partition (None = uniform strips of strip_height rows)."""
        starts = (u16 * (world_size + 1))(*strip_starts) if strip_starts is not None else None
        if arenas is not None:
            arr = (C.c_void_p * world_size)(*arenas)
            r = _lib.nrdCudaConnectPeers(self._ctx, rank, world_size, None, arr, starts)
        else:
            blob = b"".join(ipc_handles)
            assert len(blob) == IPC_HANDLE_SIZE * world_size
            r = _lib.nrdCudaConnectPeers(self._ctx, rank, world_size, blob, None, starts)
        self._check("nrdCudaConnectPeers", r)
        self.world_size = world_size

    def barrier(self, stream=0):
        self._check("nrdCudaBarrier", _lib.nrdCudaBarrier(self._ctx, C.c_void_p(stream)))

    def repartition(self, strip_starts, stream=0):
        """Collective between two frames: every connected rank passes the same world_size + 1 strip starts (include/nrd_b200.h).
        Afterwards get_texture / copy address the new rows of this rank."""
        if self.world_size is not None and len(strip_starts) != self.world_size + 1:  # the library reads world_size + 1 entries
            raise ValueError("%d strip starts for a world of %d: give world_size + 1" % (len(strip_starts), self.world_size))
        starts = (u16 * len(strip_starts))(*strip_starts)
        self._check("nrdCudaRepartition", _lib.nrdCudaRepartition(self._ctx, starts, C.c_void_p(stream)))
        viewz = self.get_texture(ResourceType.IN_VIEWZ)  # a full-resolution texture: its rows are the strip
        self.strip = (viewz.firstRow, viewz.firstRow + viewz.rowsNum)

    def synchronize(self, stream=0):
        self._check("nrdCudaSynchronize", _lib.nrdCudaSynchronize(self._ctx, C.c_void_p(stream)))

    def set_timing(self, enable):
        self._check("nrdCudaSetTiming", _lib.nrdCudaSetTiming(self._ctx, 1 if enable else 0))

    def get_timing(self):
        """(kernel_ms, exchange_ms) lists of the dispatches executed since the last call (timing must be on)."""
        k, x, n = (C.c_float * 64)(), (C.c_float * 64)(), C.c_uint32(0)
        self._check("nrdCudaGetTiming", _lib.nrdCudaGetTiming(self._ctx, k, x, 64, C.byref(n)))
        return list(k[:n.value]), list(x[:n.value])

    def execute_raw(self, raw_dispatch_ptr, stream=0):
        self._check("nrdCudaExecuteDispatch", _lib.nrdCudaExecuteDispatch(self._ctx, raw_dispatch_ptr, C.c_void_p(stream)))

    def denoise(self, identifiers, stream=0):
        ids = (u32 * len(identifiers))(*identifiers)
        n = u32(0)
        self._check("nrdCudaDenoise", _lib.nrdCudaDenoise(self._ctx, ids, len(identifiers), C.c_void_p(stream), C.byref(n)))
        return n.value


def launch_count():
    return int(_lib.nrdCudaGetLaunchCount())
