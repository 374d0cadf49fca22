"""nrdCudaSetUserTextureArray at the boundary, without a device: a null context or a null array is refused before any CUDA call."""
import ctypes as C


def test_set_user_texture_array_refuses_a_null_context_or_array():
    from raytracingdenoiser_b200 import nrd
    lib = C.CDLL(nrd.library_path())
    lib.nrdCudaSetUserTextureArray.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32]
    lib.nrdCudaSetUserTextureArray.restype = C.c_uint32
    mv, fmt = int(nrd.ResourceType.IN_MV), int(nrd.Format.RGBA16_SFLOAT)
    assert lib.nrdCudaSetUserTextureArray(None, mv, None, fmt) == nrd.Result.INVALID_ARGUMENT
    assert lib.nrdCudaSetUserTextureArray(None, mv, C.c_void_p(0x1000), fmt) == nrd.Result.INVALID_ARGUMENT
    assert "nrdCudaSetUserTextureArray" in nrd.EXPORTED_SYMBOLS
