"""User textures bound as CUDA arrays (nrdCudaSetUserTextureArray), the binding an application uses for an imported Vulkan / D3D12
image.  The arrays are made with the driver API (raytracingdenoiser_b200/cuda_arrays.py: cuArray3DCreate / cuMipmappedArrayCreate with
CUDA_ARRAY3D_SURFACE_LDST, filled and read with cuMemcpy2D): a CUarray is a cudaArray_t, so no graphics API is needed.

Every comparison runs a second context on the same seeded frames with every texture bound by pointer: after every frame each
OUT_* texture and IN_MV (which the frame-0 clear zeroes and REBLUR TemporalStabilization patches with
isBaseColorMetalnessAvailable) must hold the same bytes in the array as in the pointer-bound texture."""
import ctypes as C

import pytest

from raytracingdenoiser_b200.cuda_arrays import LAYERED, SURFACE_LDST, CudaArray

pytestmark = pytest.mark.gpu

W, H = 250, 141
FRAMES = 7
RESTART_AT = 4
ALL_OPTIONAL_INPUTS = {"isHistoryConfidenceAvailable": True, "isDisocclusionThresholdMixAvailable": True, "isBaseColorMetalnessAvailable": True}
CASES = [("REBLUR_DIFFUSE_SPECULAR", ALL_OPTIONAL_INPUTS), ("RELAX_DIFFUSE_SPECULAR", ALL_OPTIONAL_INPUTS),
         ("SIGMA_SHADOW_TRANSLUCENCY", None), ("REFERENCE", None)]


def _bytes(t):
    import torch
    return t.contiguous().view(-1).view(torch.uint8)


def _frames(den, w, h, frames=FRAMES):
    from raytracingdenoiser_b200 import harness, scene
    sc = scene.Scene(w, h)
    return [sc.frame(f, harness.radiance_mode(den)) for f in range(frames)]


def _settings(fr, w, h, f, common):
    from raytracingdenoiser_b200 import harness, nrd
    c = dict(common or {})
    if f == RESTART_AT:
        c["accumulationMode"] = int(nrd.AccumulationMode.RESTART)
    return harness.make_common_settings(fr, w, h, f, common=c)


class Bound(object):
    """One context whose user textures are bound by pointer (torch tensors) or by array, one type at a time, rebindable."""

    def __init__(self, den, w, h, common, formats=None, pad=(0, 0)):
        import torch
        from raytracingdenoiser_b200 import harness, nrd
        self.den, self.w, self.h, self.common, self.formats, self.pad = den, w, h, common, formats or {}, pad
        self.inst = nrd.Instance([(0, den)])
        self.ctx = nrd.CudaContext(self.inst, w, h)
        self.names = harness.denoiser_resources(den, common)
        self.tensors, self.arrays, self.guards = {}, {}, {}
        self.stream = torch.cuda.current_stream(torch.device("cuda", 0)).cuda_stream

    def fmt(self, name):
        from raytracingdenoiser_b200 import harness
        return self.formats.get(name, harness.user_format(self.den, name))

    def _content(self, name):
        """what the texture holds under its present binding: a rebinding carries it over, as an application that moves a
        texture would (the passes use the outputs as scratch, and texels they skip keep earlier frames' values)"""
        if name in self.arrays:
            _, dtype, ch = self.fmt(name)
            return self.arrays[name].download(dtype, ch)[:self.h, :self.w].clone()
        return self.tensors[name].clone() if name in self.tensors else None

    def bind_pointer(self, name):
        import torch
        from raytracingdenoiser_b200 import nrd
        fmt, dtype, ch = self.fmt(name)
        t = torch.zeros((self.h, self.w, ch) if ch > 1 else (self.h, self.w), dtype=dtype, device="cuda:0")
        old = self._content(name)
        if old is not None:
            t.copy_(old)
        self.ctx.set_user_texture(getattr(nrd.ResourceType, name), t.data_ptr(), t.stride(0) * t.element_size(), fmt)
        self._drop_array(name)
        self.tensors[name] = t

    def bind_array(self, name, mipmapped=False):
        """An array `pad` texels wider and taller than the resource, the texels beyond it filled with 0xA5 bytes, which no frame may change."""
        import torch
        from raytracingdenoiser_b200 import nrd
        fmt, dtype, ch = self.fmt(name)
        a = CudaArray(fmt, self.w + self.pad[0], self.h + self.pad[1], mipmapped=mipmapped)
        fill = torch.full((a.height, a.width * a.bpt), 0xA5, dtype=torch.uint8, device="cuda:0")
        fill[:self.h, :self.w * a.bpt] = 0
        a.upload(fill.view(dtype).view((a.height, a.width, ch) if ch > 1 else (a.height, a.width)))
        old = self._content(name)
        if old is not None:
            a.upload(old)
        self.ctx.set_user_texture_array(getattr(nrd.ResourceType, name), a.handle.value, fmt)
        self._drop_array(name)
        self.tensors.pop(name, None)
        self.arrays[name] = a
        self.guards[name] = fill

    def _drop_array(self, name):
        if name in self.arrays:
            self.arrays.pop(name).destroy()
            self.guards.pop(name)

    def set_inputs(self, fr):
        for name in self.names:
            if not name.startswith("IN_"):
                continue
            dtype = self.fmt(name)[1]
            if name in self.arrays:
                self.arrays[name].upload(fr[name].to(dtype))
            else:
                self.tensors[name].copy_(fr[name].to(dtype))

    def denoise(self, cs):
        self.inst.set_common_settings(cs)
        self.ctx.denoise([0], stream=self.stream)

    def dispatch_loop(self, cs):
        self.inst.set_common_settings(cs)
        r, raw, n = self.inst.get_compute_dispatches_raw([0])
        assert r == 0
        for i in range(n):
            self.ctx.execute_raw(C.byref(raw[i]), self.stream)

    def state(self):
        """OUT_* and IN_MV as (h, w[, c]) tensors; the texels of an array beyond the resource checked unchanged"""
        import torch
        torch.cuda.synchronize()
        out = {}
        for name in self.names:
            if not (name.startswith("OUT_") or name == "IN_MV"):
                continue
            if name in self.arrays:
                a = self.arrays[name]
                _, dtype, ch = self.fmt(name)
                full = a.download(dtype, ch)
                raw = _bytes(full).view(a.height, a.width * a.bpt)
                mask = torch.ones_like(raw, dtype=torch.bool)
                mask[:self.h, :self.w * a.bpt] = False
                assert torch.equal(raw[mask], self.guards[name][mask]), "%s: a texel beyond the resource size changed" % name
                out[name] = full[:self.h, :self.w]
            else:
                out[name] = self.tensors[name]
        return out

    def destroy(self):
        self.ctx.destroy()
        self.inst.destroy()
        for a in self.arrays.values():
            a.destroy()


def _compare(f, got, want):
    assert set(got) == set(want)
    for name in want:
        assert torch_equal_bytes(got[name], want[name]), "frame %d: %s differs from the pointer-bound context" % (f, name)


def torch_equal_bytes(a, b):
    import torch
    return torch.equal(_bytes(a), _bytes(b))


def _run_pair(den, w, h, common, bind, formats=None, rebind=None, loop=False, pad=(0, 0)):
    """Runs a pointer-bound context and a context bound by `bind(ctx)` on the same frames and compares them after every frame.
    rebind(ctx, f): called before frame f.  loop: the second context runs the nrdCudaExecuteDispatch loop instead of nrdCudaDenoise."""
    rw, rh = (common or {}).get("resourceSize", (w, h))
    frs = _frames(den, rw, rh)
    ref, other = Bound(den, rw, rh, common, formats), Bound(den, rw, rh, common, formats, pad=pad)
    try:
        for name in ref.names:
            ref.bind_pointer(name)
        bind(other)
        for f, fr in enumerate(frs):
            if rebind:
                rebind(other, f)
            cs = _settings(fr, rw, rh, f, common)
            for b in (ref, other):
                b.set_inputs(fr)
            ref.denoise(cs)
            (other.dispatch_loop if loop else other.denoise)(cs)
            want = ref.state()
            _compare(f, other.state(), want)
        assert any(float(t.float().abs().sum()) > 0 for k, t in want.items() if k.startswith("OUT_"))
    finally:
        ref.destroy()
        other.destroy()


def _all_arrays(b):
    for i, name in enumerate(b.names):
        b.bind_array(name, mipmapped=i % 2 == 1)


@pytest.mark.parametrize("denoiser_name,common", CASES, ids=[c[0] for c in CASES])
def test_array_bindings_give_the_pointer_result(denoiser_name, common):
    """Every user texture by array (every second one as level 0 of a mipmapped array), arrays larger than the resource: frame 0,
    a RESTART at frame 4."""
    from raytracingdenoiser_b200 import nrd
    _run_pair(getattr(nrd.Denoiser, denoiser_name), W, H, common, _all_arrays, pad=(7, 5))


@pytest.mark.parametrize("denoiser_name,common", CASES[:2], ids=[c[0] for c in CASES[:2]])
def test_array_bindings_under_dynamic_resolution(denoiser_name, common):
    """Arrays at resourceSize, a smaller rect at a non-zero rectOrigin: the guide inputs are read through the rect-origin view of
    their shadows."""
    from raytracingdenoiser_b200 import nrd
    c = dict(common or {}, resourceSize=(W, H), resourceSizePrev=(W, H), rectSize=(W - 37, H - 21), rectSizePrev=(W - 37, H - 21),
             rectOrigin=(13, 8))
    _run_pair(getattr(nrd.Denoiser, denoiser_name), W, H, c, _all_arrays)


def test_array_bindings_in_a_wider_format():
    """RGBA32_SFLOAT radiance in and out and R16_SFLOAT viewZ, by array against the same formats by pointer."""
    import torch
    from raytracingdenoiser_b200 import nrd
    wide = (nrd.Format.RGBA32_SFLOAT, torch.float32, 4)
    formats = {"IN_DIFF_RADIANCE_HITDIST": wide, "IN_SPEC_RADIANCE_HITDIST": wide, "OUT_DIFF_RADIANCE_HITDIST": wide,
               "IN_VIEWZ": (nrd.Format.R16_SFLOAT, torch.float16, 1)}
    _run_pair(nrd.Denoiser.REBLUR_DIFFUSE_SPECULAR, W, H, ALL_OPTIONAL_INPUTS, _all_arrays, formats=formats)


def test_mixed_bindings_and_rebinding_between_frames():
    """Half the textures by pointer, half by array; IN_VIEWZ goes from pointer to array and back, OUT_SPEC_RADIANCE_HITDIST from
    array to pointer and back, between frames."""
    from raytracingdenoiser_b200 import nrd

    def bind(b):
        for i, name in enumerate(b.names):
            if name == "OUT_SPEC_RADIANCE_HITDIST" or (name != "IN_VIEWZ" and i % 2 == 0):
                b.bind_array(name)
            else:
                b.bind_pointer(name)

    def rebind(b, f):
        if f == 2:
            b.bind_array("IN_VIEWZ", mipmapped=True)
            b.bind_pointer("OUT_SPEC_RADIANCE_HITDIST")
        elif f == 5:
            b.bind_pointer("IN_VIEWZ")
            b.bind_array("OUT_SPEC_RADIANCE_HITDIST")

    _run_pair(nrd.Denoiser.REBLUR_DIFFUSE_SPECULAR, W, H, ALL_OPTIONAL_INPUTS, bind, rebind=rebind)


@pytest.mark.parametrize("denoiser_name,common", CASES[:2], ids=[c[0] for c in CASES[:2]])
def test_dispatch_loop_gives_the_denoise_result(denoiser_name, common):
    """nrdCudaExecuteDispatch converts what each dispatch reads before it and writes back what it writes after it; with every
    texture an array the loop ends every frame with the bytes of the pointer-bound nrdCudaDenoise, IN_MV included."""
    from raytracingdenoiser_b200 import nrd
    _run_pair(getattr(nrd.Denoiser, denoiser_name), W, H, common, _all_arrays, loop=True)


def test_refusals():
    import torch
    from raytracingdenoiser_b200 import nrd
    den = nrd.Denoiser.REBLUR_DIFFUSE_SPECULAR
    inst = nrd.Instance([(0, den)])
    ctx = nrd.CudaContext(inst, 64, 48)
    made = []

    def array(fmt, w=64, h=48, **kw):
        made.append(CudaArray(fmt, w, h, **kw))
        return made[-1].handle.value

    def refused(result, rtype, handle, fmt):
        with pytest.raises(nrd.NrdError) as e:
            ctx.set_user_texture_array(rtype, handle, fmt)
        assert e.value.result == result, str(e.value)
        assert "[]" not in str(e.value), "no message for %s" % e.value

    R, F, T = nrd.Result, nrd.Format, nrd.ResourceType
    try:
        refused(R.INVALID_ARGUMENT, T.IN_VIEWZ, None, F.R32_SFLOAT)
        refused(R.INVALID_ARGUMENT, T.IN_VIEWZ, array(F.R32_SFLOAT, w=63), F.R32_SFLOAT)
        refused(R.INVALID_ARGUMENT, T.IN_VIEWZ, array(F.R32_SFLOAT, h=47), F.R32_SFLOAT)
        refused(R.UNSUPPORTED, T.IN_VIEWZ, array(F.R32_SFLOAT, depth=2, flags=SURFACE_LDST | LAYERED), F.R32_SFLOAT)
        refused(R.UNSUPPORTED, T.IN_VIEWZ, array(F.R32_SFLOAT, depth=2), F.R32_SFLOAT)
        refused(R.UNSUPPORTED, T.IN_VIEWZ, array(F.R32_SFLOAT, flags=0), F.R32_SFLOAT)
        refused(R.UNSUPPORTED, T.IN_VIEWZ, array(F.R16_SFLOAT), F.R32_SFLOAT)           # element size
        refused(R.UNSUPPORTED, T.IN_VIEWZ, array(F.RGBA8_UNORM), F.RGBA8_UNORM)         # UNORM for a float format
        refused(R.UNSUPPORTED, T.IN_DIFF_SH0, array(F.RGBA16_SFLOAT), F.RGBA16_SFLOAT)  # no supported denoiser reads it
        ctx.set_user_texture_array(T.IN_VIEWZ, array(F.R32_SFLOAT, w=100, h=60), F.R32_SFLOAT)  # larger is fine
        info = ctx.get_texture(T.IN_VIEWZ)
        assert (info.width, info.height, info.format) == (64, 48, F.R32_SFLOAT)
        strip_inst = nrd.Instance([(0, den)])
        strip = nrd.CudaContext(strip_inst, 64, 48, strip=(0, 48), strip_height=48)
        try:
            for bind in (lambda: strip.set_user_texture(T.IN_VIEWZ, torch.zeros(48, 64, device="cuda:0").data_ptr(), 256, F.R32_SFLOAT),
                         lambda: strip.set_user_texture_array(T.IN_VIEWZ, array(F.R32_SFLOAT), F.R32_SFLOAT)):
                with pytest.raises(nrd.NrdError) as e:
                    bind()
                assert e.value.result == R.UNSUPPORTED and "strip mode" in str(e.value)
        finally:
            strip.destroy()
            strip_inst.destroy()
    finally:
        ctx.destroy()
        inst.destroy()
        for a in made:
            a.destroy()


def test_rebinding_releases_the_shadow():
    """200 rebinds of a 2048 x 1024 RGBA16 texture (16 MiB shadow each), alternately by array and by pointer: the device memory
    free afterwards is what it was after the first binding."""
    import torch
    from raytracingdenoiser_b200 import nrd
    w, h = 2048, 1024
    inst = nrd.Instance([(0, nrd.Denoiser.REFERENCE)])
    ctx = nrd.CudaContext(inst, w, h)
    a = CudaArray(nrd.Format.RGBA16_SFLOAT, w, h)
    t = torch.zeros((h, w, 4), dtype=torch.float16, device="cuda:0")
    try:
        ctx.set_user_texture_array(nrd.ResourceType.IN_SIGNAL, a.handle.value, nrd.Format.RGBA16_SFLOAT)
        torch.cuda.synchronize()
        before = torch.cuda.mem_get_info(0)[0]
        for i in range(200):
            if i % 4 == 3:
                ctx.set_user_texture(nrd.ResourceType.IN_SIGNAL, t.data_ptr(), w * 8, nrd.Format.RGBA16_SFLOAT)
            else:
                ctx.set_user_texture_array(nrd.ResourceType.IN_SIGNAL, a.handle.value, nrd.Format.RGBA16_SFLOAT)
        torch.cuda.synchronize()
        after = torch.cuda.mem_get_info(0)[0]
        assert before - after < 64 << 20, "%.0f MiB of device memory not returned after 200 rebinds" % ((before - after) / 2.0 ** 20)
    finally:
        ctx.destroy()
        inst.destroy()
        a.destroy()
