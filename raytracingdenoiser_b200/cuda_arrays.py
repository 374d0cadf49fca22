"""2D CUDA arrays made with the driver API through ctypes (libcuda.so), for the tests and tools of nrdCudaSetUserTextureArray.

A CUarray is a cudaArray_t, so an array made here stands for the one an application gets from an imported Vulkan / D3D12 image
(cudaExternalMemoryGetMappedMipmappedArray + level 0) without a graphics API.  Arrays live in the primary context of device 0,
the context torch and the library use too.
"""
import ctypes as C

import torch

SURFACE_LDST, LAYERED = 0x02, 0x01  # CUDA_ARRAY3D_SURFACE_LDST, CUDA_ARRAY3D_LAYERED
_CU_AD = {"u8": 0x01, "f16": 0x10, "u32": 0x03, "f32": 0x20}  # CUarray_format
_KIND_BYTES = {"u8": 1, "f16": 2, "u32": 4, "f32": 4}
# nrd.Format name -> (element kind, channels): texels are the raw bytes of the format (packed R10G10B10A2 is one 32-bit channel)
ARRAY_FORMATS = {"R8_UNORM": ("u8", 1), "RGBA8_UNORM": ("u8", 4), "R16_SFLOAT": ("f16", 1), "RG16_SFLOAT": ("f16", 2), "RGBA16_SFLOAT": ("f16", 4),
                 "R32_SFLOAT": ("f32", 1), "RG32_SFLOAT": ("f32", 2), "RGBA32_SFLOAT": ("f32", 4), "R10_G10_B10_A2_UNORM": ("u32", 1)}


class _Desc3D(C.Structure):
    _fields_ = [("Width", C.c_size_t), ("Height", C.c_size_t), ("Depth", C.c_size_t), ("Format", C.c_int), ("NumChannels", C.c_uint),
                ("Flags", C.c_uint)]


class _Memcpy2D(C.Structure):
    _fields_ = [("srcXInBytes", C.c_size_t), ("srcY", C.c_size_t), ("srcMemoryType", C.c_int), ("srcHost", C.c_void_p), ("srcDevice", C.c_uint64),
                ("srcArray", C.c_void_p), ("srcPitch", C.c_size_t), ("dstXInBytes", C.c_size_t), ("dstY", C.c_size_t), ("dstMemoryType", C.c_int),
                ("dstHost", C.c_void_p), ("dstDevice", C.c_uint64), ("dstArray", C.c_void_p), ("dstPitch", C.c_size_t), ("WidthInBytes", C.c_size_t),
                ("Height", C.c_size_t)]


_MEMORY_DEVICE, _MEMORY_ARRAY = 2, 3  # CUmemorytype
_driver = None


def driver():
    """libcuda.so, with the primary context of device 0 current on this thread"""
    global _driver
    torch.zeros(1, device="cuda:0")
    if _driver is None:
        _driver = C.CDLL("libcuda.so.1")
    return _driver


def _ok(r, what):
    if r != 0:
        raise RuntimeError("%s -> CUresult %d" % (what, r))


class CudaArray(object):
    """A CUarray in the layout of an nrd.Format: 2D by default, level 0 of a three-level mipmapped array with mipmapped=True;
    `flags` / `depth` make the layered, 3D or non-surface arrays the library refuses."""

    def __init__(self, fmt, width, height, mipmapped=False, flags=SURFACE_LDST, depth=0):
        cu = driver()
        kind, ch = ARRAY_FORMATS[fmt.name]
        self.width, self.height, self.bpt = width, height, ch * _KIND_BYTES[kind]
        desc = _Desc3D(width, height, depth, _CU_AD[kind], ch, flags)
        self.handle, self.mip = C.c_void_p(), None
        if mipmapped:
            self.mip = C.c_void_p()
            _ok(cu.cuMipmappedArrayCreate(C.byref(self.mip), C.byref(desc), 3), "cuMipmappedArrayCreate")
            _ok(cu.cuMipmappedArrayGetLevel(C.byref(self.handle), self.mip, 0), "cuMipmappedArrayGetLevel")
        else:
            _ok(cu.cuArray3DCreate_v2(C.byref(self.handle), C.byref(desc)), "cuArray3DCreate")

    def _copy(self, t, to_array):
        assert t.is_contiguous() and t.shape[1] <= self.width and t.shape[0] <= self.height
        torch.cuda.synchronize()  # cuMemcpy2D is ordered with the legacy default stream only
        m = _Memcpy2D()
        m.WidthInBytes, m.Height = t.shape[1] * self.bpt, t.shape[0]
        if to_array:
            m.srcMemoryType, m.srcDevice, m.srcPitch = _MEMORY_DEVICE, t.data_ptr(), t.stride(0) * t.element_size()
            m.dstMemoryType, m.dstArray = _MEMORY_ARRAY, self.handle
        else:
            m.srcMemoryType, m.srcArray = _MEMORY_ARRAY, self.handle
            m.dstMemoryType, m.dstDevice, m.dstPitch = _MEMORY_DEVICE, t.data_ptr(), t.stride(0) * t.element_size()
        _ok(driver().cuMemcpy2D_v2(C.byref(m)), "cuMemcpy2D")

    def upload(self, t):
        """t: a (h, w[, c]) tensor of the format's texels (host or device), copied to texels [0, w) x [0, h)"""
        self._copy(t.to("cuda:0").contiguous(), True)

    def download(self, dtype, channels):
        """the whole array as a (height, width[, channels]) device tensor"""
        t = torch.empty((self.height, self.width, channels) if channels > 1 else (self.height, self.width), dtype=dtype, device="cuda:0")
        self._copy(t, False)
        return t

    def destroy(self):
        if self.mip is not None:
            _ok(driver().cuMipmappedArrayDestroy(self.mip), "cuMipmappedArrayDestroy")
        elif self.handle:
            _ok(driver().cuArrayDestroy(self.handle), "cuArrayDestroy")
        self.handle, self.mip = C.c_void_p(), None
