// Device-side building blocks shared by all sm_90a kernels: pitched HBM surfaces with format-exact loads/stores,
// small vector math, and the numerically "pinned" helpers.
//
// Pinned arithmetic: wherever a result feeds floor()/step() that selects WHICH texel is read (tap positions,
// reprojection footprints) the computation is written with explicit round-to-nearest IEEE intrinsics (__fmul_rn,
// __fadd_rn, __fdiv_rn, __fsqrt_rn; never contracted to FMA) in the same operation order as the CPU oracle, so both
// pick the same texel.  Everything else is free to use FMA contraction and fast intrinsics (results agree to ~1e-6).
#pragma once
// The kernels are built twice from the same sources: the one-GPU build (-DNRD_B200_NO_STRIPS, namespace nrdb200_single)
// addresses surfaces with a plain pitch computation; the strip build (namespace nrdb200) adds the ghost-row / peer lookup
// of the multi-GPU mode.  Keeping that lookup out of the one-GPU kernels is worth ~30 % of their run time (registers,
// code size and a divergent branch around every load).
#if defined(NRD_B200_NO_STRIPS)
#define nrdb200 nrdb200_single
#endif
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "surf.h"

// Kernel launch of a pass.  With p.preloadOnly the kernel is only loaded: CUDA loads kernels lazily on first launch, and that
// load waits for the device to go idle -- which never happens while a StripBarrierKernel of this process spins for a peer
// whose next kernel is the one being loaded.  Strip-mode contexts therefore preload their kernels at creation.
#define NRD_B200_LAUNCH(p, grid, block, args, ...)                              \
    do                                                                          \
    {                                                                           \
        if ((p).preloadOnly)                                                    \
        {                                                                       \
            cudaFuncAttributes fa_;                                             \
            cudaError_t pe_ = cudaFuncGetAttributes(&fa_, __VA_ARGS__);         \
            if (pe_ != cudaSuccess) return pe_;                                 \
        }                                                                       \
        else                                                                    \
            __VA_ARGS__<<<grid, block, 0, (p).stream>>>(args);                  \
    } while (0)

namespace nrdb200
{
using namespace nrdb200_abi;

// Host side: reads the bindings of a dispatch in the order its recipe binds them (recipes_*.cpp).  Next(false) is a binding the
// pass does not have (the other signal of a one-signal denoiser): a null surface, and the next binding stays next.  A launcher
// checks Complete() before it launches: a dispatch that binds more or fewer textures than the pass reads is refused.  Preload
// launches bind nothing.
struct Bindings
{
    const PassLaunch& p;
    uint32_t read = 0;
    explicit Bindings(const PassLaunch& launch) : p(launch) {}
    Surf Next(bool present = true)
    {
        if (!present) return Surf{};
        const uint32_t i = read++;
        return i < p.texNum ? p.tex[i] : Surf{};
    }
    bool Complete() const { return p.preloadOnly || read == p.texNum; }
};

// ---------------------------------------------------------------------------------------------
// Surfaces (surf.h)
// ---------------------------------------------------------------------------------------------
#if !defined(NRD_B200_NO_STRIPS)
// strip geometry, one table per context slot (surf.h)
static __constant__ PeerTable g_peerTable[kMaxPeerSlots];
// stream == nullptr: `table` is host memory, copied before the call returns (nrdCudaConnectPeers); else `table` is device memory,
// copied in order on *stream (nrdCudaRepartition: the kernels queued before the copy still read the old table)
static inline cudaError_t SetPeerTableThisTU(int slot, const PeerTable* table, const cudaStream_t* stream)
{
    const size_t offset = sizeof(PeerTable) * (size_t)slot;
    return stream ? cudaMemcpyToSymbolAsync(g_peerTable, table, sizeof(PeerTable), offset, cudaMemcpyDeviceToDevice, *stream)
                  : cudaMemcpyToSymbol(g_peerTable, table, sizeof(PeerTable), offset);
}
// rare path: the row is beyond the ghost rows, fetch it from its owner (callers clamp y to [0, h))
// (inlined on purpose: a real call gives the kernels a stack frame, and the first launch of a kernel that needs a bigger
// stack makes the driver wait for every running kernel -- including a spinning StripBarrierKernel of another context)
static __device__ __forceinline__ const uint8_t* PeerRow(const Surf& s, int y)
{
    const PeerTable& t = g_peerTable[s.peerSlot];
    const int yFull = y << s.rowShift;
    int owner = 0;
#pragma unroll
    for (int k = 1; k < kMaxPeers; k++) owner += yFull >= t.start[k] ? 1 : 0;
    return s.base + t.delta[owner] + (size_t)(y - (t.start[owner] >> s.rowShift) + s.halo) * s.pitch;
}
#endif

template <class T> __device__ __forceinline__ const T* TexelPtr(const Surf& s, int x, int y)
{
#if defined(NRD_B200_NO_STRIPS)
    return reinterpret_cast<const T*>(s.base + (size_t)y * s.pitch) + x; // the whole texture is local: ly0 == 0 (arena.cu Arena::ToSurf)
#else
    const int ly = y - s.ly0;
    if (s.stripRows != 0 && (unsigned)ly >= s.lrows) return reinterpret_cast<const T*>(PeerRow(s, y)) + x;
    return reinterpret_cast<const T*>(s.base + (size_t)ly * s.pitch) + x;
#endif
}
// The owner lookup above costs a divergent branch and ~10 instructions of code around EVERY load.  Kernels avoid it where the
// row is known to be local: Near(s) is a view of the surface whose loads skip the lookup (stripRows = 0 is a compile-time
// constant after inlining) -- legal for the centre pixel and its fixed small neighbourhoods (the halo is >= 16 rows), and for
// whole footprints / taps after one RowsLocal() test: `if (RowsLocal(s, y0, y1)) f(Near(s)); else f(s);`.
__device__ __forceinline__ Surf Near(const Surf& s)
{
#if defined(NRD_B200_NO_STRIPS)
    return s;
#else
    Surf r = s;
    r.stripRows = 0;
    return r;
#endif
}
// rows [ya, yb] (inclusive, inside the frame) are all held by this GPU (own strip or ghost rows)
__device__ __forceinline__ bool RowsLocal(const Surf& s, int ya, int yb)
{
#if defined(NRD_B200_NO_STRIPS)
    return true;
#else
    return (unsigned)(ya - s.ly0) < s.lrows && (unsigned)(yb - s.ly0) < s.lrows;
#endif
}
// One owner lookup for several surfaces of the same geometry (full-resolution pool / user / guide surfaces share strip rows, halo and
// the peers' arena deltas): RefRow() resolves row y once, TexelAt() addresses any of those surfaces with it.
struct RowRef
{
    long long delta; // 0 = held locally (own rows or ghost rows), else the owner's arena delta
    int row;         // row index inside the holder's copy of the surface
};
__device__ __forceinline__ RowRef RefRow(const Surf& s, int y)
{
#if defined(NRD_B200_NO_STRIPS)
    (void)s;
    return {0, y};
#else
    const int ly = y - s.ly0;
    if (s.stripRows == 0 || (unsigned)ly < s.lrows) return {0, ly};
    const PeerTable& t = g_peerTable[s.peerSlot];
    const int yFull = y << s.rowShift;
    int owner = 0;
#pragma unroll
    for (int k = 1; k < kMaxPeers; k++) owner += yFull >= t.start[k] ? 1 : 0;
    return {t.delta[owner], y - (t.start[owner] >> s.rowShift) + s.halo};
#endif
}
template <class T> __device__ __forceinline__ const T* TexelAt(const Surf& s, RowRef r, int x)
{
    return reinterpret_cast<const T*>(s.base + r.delta + (size_t)r.row * s.pitch) + x;
}
template <class T> __device__ __forceinline__ T* TexelPtrRW(const Surf& s, int x, int y)
{
#if defined(NRD_B200_NO_STRIPS)
    return reinterpret_cast<T*>(s.base + (size_t)y * s.pitch) + x;
#else
    return reinterpret_cast<T*>(s.base + (size_t)(y - s.ly0) * s.pitch) + x;
#endif
}
__device__ __forceinline__ bool Inside(const Surf& s, int x, int y) { return (unsigned)x < (unsigned)s.w && (unsigned)y < (unsigned)s.h; }

// ---------------------------------------------------------------------------------------------
// Vector math (only what the kernels use)
// ---------------------------------------------------------------------------------------------
struct f2 { float x, y; };
struct f3 { float x, y, z; };
struct f4 { float x, y, z, w; };

__device__ __forceinline__ f2 mk2(float x, float y) { return {x, y}; }
__device__ __forceinline__ f3 mk3(float x, float y, float z) { return {x, y, z}; }
__device__ __forceinline__ f3 mk3(float v) { return {v, v, v}; }
__device__ __forceinline__ f4 mk4(float x, float y, float z, float w) { return {x, y, z, w}; }
__device__ __forceinline__ f4 mk4(float v) { return {v, v, v, v}; }
__device__ __forceinline__ f4 mk4(f3 a, float w) { return {a.x, a.y, a.z, w}; }
__device__ __forceinline__ f3 xyz(f4 a) { return {a.x, a.y, a.z}; }

__device__ __forceinline__ f2 operator+(f2 a, f2 b) { return {a.x + b.x, a.y + b.y}; }
__device__ __forceinline__ f2 operator-(f2 a, f2 b) { return {a.x - b.x, a.y - b.y}; }
__device__ __forceinline__ f2 operator*(f2 a, f2 b) { return {a.x * b.x, a.y * b.y}; }
__device__ __forceinline__ f2 operator*(f2 a, float b) { return {a.x * b, a.y * b}; }
__device__ __forceinline__ f3 operator+(f3 a, f3 b) { return {a.x + b.x, a.y + b.y, a.z + b.z}; }
__device__ __forceinline__ f3 operator-(f3 a, f3 b) { return {a.x - b.x, a.y - b.y, a.z - b.z}; }
__device__ __forceinline__ f3 operator-(f3 a) { return {-a.x, -a.y, -a.z}; }
__device__ __forceinline__ f3 operator*(f3 a, f3 b) { return {a.x * b.x, a.y * b.y, a.z * b.z}; }
__device__ __forceinline__ f3 operator*(f3 a, float b) { return {a.x * b, a.y * b, a.z * b}; }
__device__ __forceinline__ f4 operator+(f4 a, f4 b) { return {a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w}; }
__device__ __forceinline__ f4 operator-(f4 a, f4 b) { return {a.x - b.x, a.y - b.y, a.z - b.z, a.w - b.w}; }
__device__ __forceinline__ f4 operator*(f4 a, f4 b) { return {a.x * b.x, a.y * b.y, a.z * b.z, a.w * b.w}; }
__device__ __forceinline__ f4 operator*(f4 a, float b) { return {a.x * b, a.y * b, a.z * b, a.w * b}; }
__device__ __forceinline__ float dot(f2 a, f2 b) { return a.x * b.x + a.y * b.y; }
__device__ __forceinline__ float dot(f3 a, f3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
__device__ __forceinline__ float dot(f4 a, f4 b) { return a.x * b.x + a.y * b.y + a.z * b.z + a.w * b.w; }
__device__ __forceinline__ float length(f2 a) { return sqrtf(dot(a, a)); }
__device__ __forceinline__ float length(f3 a) { return sqrtf(dot(a, a)); }
__device__ __forceinline__ f3 normalize(f3 a) { return a * rsqrtf(dot(a, a)); }
__device__ __forceinline__ f3 cross(f3 a, f3 b) { return {a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x}; }
__device__ __forceinline__ f3 reflect(f3 i, f3 n) { return i - n * (2.0f * dot(i, n)); }
__device__ __forceinline__ float saturate(float x) { return __saturatef(x); } // NaN -> 0, like HLSL
// Saturating arithmetic as ONE instruction.  nvcc does not fold __saturatef() (cvt.sat) or fabsf() into the producing FADD / FFMA
// when -ftz is on: saturate(1 - |x|) compiles to three instructions (FADD |x|, FADD 1 - x, FADD.SAT) -- and these kernels are
// issue-bound.  Spelled as PTX the .sat and the |.| / - operand modifiers land on the arithmetic instruction itself.
__device__ __forceinline__ float SatFma(float a, float b, float c)
{
    float r;
    asm("fma.rn.sat.ftz.f32 %0, %1, %2, %3;" : "=f"(r) : "f"(a), "f"(b), "f"(c));
    return r;
}
__device__ __forceinline__ float SatAdd(float a, float b)
{
    float r;
    asm("add.sat.ftz.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
    return r;
}
__device__ __forceinline__ float SatMul(float a, float b)
{
    float r;
    asm("mul.sat.ftz.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
    return r;
}
__device__ __forceinline__ float OneMinusSat(float x) { return SatFma(x, -1.0f, 1.0f); }       // saturate(1 - x)
__device__ __forceinline__ float OneMinusAbsSat(float x) { return SatFma(fabsf(x), -1.0f, 1.0f); } // saturate(1 - |x|)
__device__ __forceinline__ float lerpf(float a, float b, float t) { return a + (b - a) * t; }
__device__ __forceinline__ f2 lerp2(f2 a, f2 b, float t) { return {lerpf(a.x, b.x, t), lerpf(a.y, b.y, t)}; }
__device__ __forceinline__ f3 lerp3(f3 a, f3 b, float t) { return {lerpf(a.x, b.x, t), lerpf(a.y, b.y, t), lerpf(a.z, b.z, t)}; }
__device__ __forceinline__ f4 lerp4(f4 a, f4 b, float t) { return {lerpf(a.x, b.x, t), lerpf(a.y, b.y, t), lerpf(a.z, b.z, t), lerpf(a.w, b.w, t)}; }
__device__ __forceinline__ float stepf(float a, float x) { return x >= a ? 1.0f : 0.0f; }
__device__ __forceinline__ float clampf(float x, float a, float b) { return fminf(fmaxf(x, a), b); }
__device__ __forceinline__ int clampi(int x, int a, int b) { return min(max(x, a), b); }

// column-major 4x4 stored as 16 floats (column k = m[4k .. 4k+3])
// pinned mul(M, (p, 1)): ((c0*x + c1*y) + c2*z) + c3, products and sums individually rounded
__device__ __forceinline__ float PinnedRow(const float* m, int r, float x, float y, float z)
{
    float s = __fadd_rn(__fmul_rn(m[0 + r], x), __fmul_rn(m[4 + r], y));
    s = __fadd_rn(s, __fmul_rn(m[8 + r], z));
    return __fadd_rn(s, __fmul_rn(m[12 + r], 1.0f));
}
// rotation by the upper 3x3:  c0*x + c1*y + c2*z   (same order, pinned)
__device__ __forceinline__ f3 PinnedRotate(const float* m, f3 v)
{
    f3 r;
    r.x = __fadd_rn(__fadd_rn(__fmul_rn(m[0], v.x), __fmul_rn(m[4], v.y)), __fmul_rn(m[8], v.z));
    r.y = __fadd_rn(__fadd_rn(__fmul_rn(m[1], v.x), __fmul_rn(m[5], v.y)), __fmul_rn(m[9], v.z));
    r.z = __fadd_rn(__fadd_rn(__fmul_rn(m[2], v.x), __fmul_rn(m[6], v.y)), __fmul_rn(m[10], v.z));
    return r;
}
// rotation by the transpose of the upper 3x3: dot(column k, v), pinned left-to-right
__device__ __forceinline__ float PinnedDot3(float ax, float ay, float az, f3 v)
{
    return __fadd_rn(__fadd_rn(__fmul_rn(ax, v.x), __fmul_rn(ay, v.y)), __fmul_rn(az, v.z));
}
__device__ __forceinline__ f3 PinnedRotateInverse(const float* m, f3 v)
{
    return {PinnedDot3(m[0], m[1], m[2], v), PinnedDot3(m[4], m[5], m[6], v), PinnedDot3(m[8], m[9], m[10], v)};
}
__device__ __forceinline__ f3 RotateInverse(const float* m, f3 v)
{
    return {m[0] * v.x + m[1] * v.y + m[2] * v.z, m[4] * v.x + m[5] * v.y + m[6] * v.z, m[8] * v.x + m[9] * v.y + m[10] * v.z};
}
__device__ __forceinline__ f3 Rotate(const float* m, f3 v)
{
    return {m[0] * v.x + m[4] * v.y + m[8] * v.z, m[1] * v.x + m[5] * v.y + m[9] * v.z, m[2] * v.x + m[6] * v.y + m[10] * v.z};
}

// ---------------------------------------------------------------------------------------------
// Format-exact texel access.  Loads use the read-only path; OOB loads return 0 and OOB stores are dropped
// only where a kernel asks for it explicitly (most kernels clamp coordinates first).
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ f4 UnpackHalf4(uint2 v)
{
    __half2 a = *reinterpret_cast<__half2*>(&v.x), b = *reinterpret_cast<__half2*>(&v.y);
    float2 fa = __half22float2(a), fb = __half22float2(b);
    return {fa.x, fa.y, fb.x, fb.y};
}
__device__ __forceinline__ uint2 PackHalf4(f4 v)
{
    __half2 a = __floats2half2_rn(v.x, v.y), b = __floats2half2_rn(v.z, v.w);
    uint2 r;
    r.x = *reinterpret_cast<unsigned*>(&a);
    r.y = *reinterpret_cast<unsigned*>(&b);
    return r;
}
__device__ __forceinline__ f4 LoadRGBA16F(const Surf& s, int x, int y) { return UnpackHalf4(__ldg(TexelPtr<uint2>(s, x, y))); }
__device__ __forceinline__ void StoreRGBA16F(const Surf& s, int x, int y, f4 v) { *TexelPtrRW<uint2>(s, x, y) = PackHalf4(v); }
__device__ __forceinline__ float LoadR16F(const Surf& s, int x, int y) { return __half2float(__ushort_as_half(__ldg(TexelPtr<unsigned short>(s, x, y)))); }
__device__ __forceinline__ void StoreR16F(const Surf& s, int x, int y, float v) { *TexelPtrRW<unsigned short>(s, x, y) = __half_as_ushort(__float2half_rn(v)); }
__device__ __forceinline__ f4 LoadRGBA32F(const Surf& s, int x, int y)
{
    float4 v = __ldg(TexelPtr<float4>(s, x, y));
    return {v.x, v.y, v.z, v.w};
}
__device__ __forceinline__ void StoreRGBA32F(const Surf& s, int x, int y, f4 v) { *TexelPtrRW<float4>(s, x, y) = make_float4(v.x, v.y, v.z, v.w); }
__device__ __forceinline__ float LoadR32F(const Surf& s, int x, int y) { return __ldg(TexelPtr<float>(s, x, y)); }
__device__ __forceinline__ void StoreR32F(const Surf& s, int x, int y, float v) { *TexelPtrRW<float>(s, x, y) = v; }
__device__ __forceinline__ unsigned LoadU32(const Surf& s, int x, int y) { return __ldg(TexelPtr<unsigned>(s, x, y)); }
__device__ __forceinline__ void StoreU32(const Surf& s, int x, int y, unsigned v) { *TexelPtrRW<unsigned>(s, x, y) = v; }
__device__ __forceinline__ unsigned LoadU16(const Surf& s, int x, int y) { return __ldg(TexelPtr<unsigned short>(s, x, y)); }
__device__ __forceinline__ void StoreU16(const Surf& s, int x, int y, unsigned v) { *TexelPtrRW<unsigned short>(s, x, y) = (unsigned short)v; }
__device__ __forceinline__ unsigned LoadU8(const Surf& s, int x, int y) { return __ldg(TexelPtr<unsigned char>(s, x, y)); }
__device__ __forceinline__ void StoreU8(const Surf& s, int x, int y, unsigned v) { *TexelPtrRW<unsigned char>(s, x, y) = (unsigned char)v; }
// UNORM: round-half-up of saturate(x) * max (D3D float -> UNORM), NaN -> 0
__device__ __forceinline__ unsigned ToUnorm(float v, float maxv) { return (unsigned)__fadd_rn(__fmul_rn(__saturatef(v), maxv), 0.5f); }
__device__ __forceinline__ float LoadR8Unorm(const Surf& s, int x, int y) { return (float)LoadU8(s, x, y) / 255.0f; }
__device__ __forceinline__ void StoreR8Unorm(const Surf& s, int x, int y, float v) { StoreU8(s, x, y, ToUnorm(v, 255.0f)); }
__device__ __forceinline__ f2 LoadRG8Unorm(const Surf& s, int x, int y)
{
    unsigned v = LoadU16(s, x, y);
    return {(float)(v & 255u) / 255.0f, (float)(v >> 8) / 255.0f};
}
__device__ __forceinline__ void StoreRG8Unorm(const Surf& s, int x, int y, f2 v) { StoreU16(s, x, y, ToUnorm(v.x, 255.0f) | (ToUnorm(v.y, 255.0f) << 8)); }
__device__ __forceinline__ f4 UnpackR10G10B10A2(unsigned v)
{
    return {(float)(v & 1023u) / 1023.0f, (float)((v >> 10) & 1023u) / 1023.0f, (float)((v >> 20) & 1023u) / 1023.0f, (float)(v >> 30) / 3.0f};
}
__device__ __forceinline__ unsigned PackR10G10B10A2(f4 v)
{
    return ToUnorm(v.x, 1023.0f) | (ToUnorm(v.y, 1023.0f) << 10) | (ToUnorm(v.z, 1023.0f) << 20) | (ToUnorm(v.w, 3.0f) << 30);
}
__device__ __forceinline__ f4 UnpackRGBA8(unsigned v)
{
    return {(float)(v & 255u) / 255.0f, (float)((v >> 8) & 255u) / 255.0f, (float)((v >> 16) & 255u) / 255.0f, (float)(v >> 24) / 255.0f};
}
__device__ __forceinline__ unsigned PackRGBA8(f4 v)
{
    return ToUnorm(v.x, 255.0f) | (ToUnorm(v.y, 255.0f) << 8) | (ToUnorm(v.z, 255.0f) << 16) | (ToUnorm(v.w, 255.0f) << 24);
}

// ---------------------------------------------------------------------------------------------
// Integer hash stream standing in for MathLib's Rng::Hash (frozen choice; bit-identical to the oracle's RngHash)
// ---------------------------------------------------------------------------------------------
struct RngHash
{
    unsigned state;
    static __device__ __forceinline__ unsigned pcg(unsigned v)
    {
        unsigned s = v * 747796405u + 2891336453u;
        unsigned w = ((s >> ((s >> 28u) + 4u)) ^ s) * 277803737u;
        return (w >> 22u) ^ w;
    }
    __device__ __forceinline__ void Initialize(int x, int y, unsigned frameIndex) { state = pcg((unsigned)x + pcg((unsigned)y + pcg(frameIndex))); }
    __device__ __forceinline__ float GetFloat()
    {
        state = pcg(state);
        return (float)(state >> 8) * (1.0f / 16777216.0f);
    }
};

} // namespace nrdb200
