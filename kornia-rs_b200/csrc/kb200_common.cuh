// kb200_common.cuh — shared host/device helpers of libkornia_b200.so (sm_90a only).
//
// Compile contract (see __graft_entry__.build): -gencode arch=compute_90a,code=sm_90a
// -fmad=false.  The reference JIT-compiles every kernel with fmad=false
// (crates/kornia-tensor/src/cuda.rs:675-718) so that `a*b + c` in kernel source rounds twice,
// exactly like the Rust CPU code; we keep that rule for the whole library and write fmaf()
// explicitly where a reference leaf is an FMA.  Division and sqrt are IEEE (nvcc defaults
// -prec-div=true -prec-sqrt=true -ftz=false).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include <cstdarg>
#include <cstdio>
#include <string>

#define KB200_BUILDING 1
#include "../../include/kornia_b200.h"

namespace kb200 {

// ── error model ─────────────────────────────────────────────────────────────────────────────
std::string& last_error_ref();
int fail(int status, const char* fmt, ...) __attribute__((format(printf, 2, 3)));
int check_launch(const char* what);  // cudaGetLastError() -> KB200_ERR_CUDA; records `what` for kb200_last_kernel()

// Developer tuning knobs (kb200_debug_set_knob): process-wide integers the launchers consult instead of the
// environment.  0 = "use the built-in choice".  Product code never needs them; sweeps and tests do.
enum Knob {
    KNOB_FR_NPX = 0, KNOB_FR_STAGES, KNOB_FR_CTAS,          // fused_rows (resize_fused.cu), tiled schedule
    KNOB_FR_ROWS,                                           // fused_rows point mode: 1 tiled, 2 full-row kernel
    KNOB_SS_STAGES, KNOB_SS_CTAS, KNOB_SS_RC,               // sep_filter_stream2 (filter.cu)
    KNOB_WARP_PF, KNOB_WARP_PATH,                           // warp.cu: prefetch rows (-1 = off); forced path (1 gather, 2 tiled, 3 stream)
    KNOB_WS_STAGES, KNOB_WS_CTAS, KNOB_WS_RC, KNOB_WS_NPX,  // warp_stream
    KNOB_RS_STAGES, KNOB_RS_CTAS, KNOB_RS_NPX,              // resize_rows_f32
    // A/B switches of the tests and tools (0 = shipped choice):
    //   a  f32 warps / remap: 3 round-2 x4 kernel, 2 the same with the shared reciprocal, 4 lean kernel general path only,
    //      5 lean kernel with STG stores, 7 lean kernel with four 1-D row copies per warp, 6 remap thread-per-pixel kernel
    //   b  u8 samplers: 1 byte taps / clamped sampler everywhere, 2 word taps in remap_u8's general path; u8 blur: 3 tile kernel
    //   c  u8 warps: 32-pixel segments per warp; u8 blur: CTAs per SM
    //   d  u8 blur: rows per chunk
    KNOB_A, KNOB_B, KNOB_C, KNOB_D,
    KNOB_COUNT
};
int knob(Knob k);

// SliceTooSmall{what,got,need} — cuda/mod.rs:104-126
inline int check_slice(const char* what, size_t got, size_t need) {
    if (got < need) return fail(KB200_ERR_SLICE_TOO_SMALL, "device slice '%s' length %zu < required %zu", what, got, need);
    return KB200_OK;
}
// check_geometry — cuda/mod.rs:182-196
inline int check_geometry(uint32_t sw, uint32_t sh, uint32_t dw, uint32_t dh, uint32_t batch) {
    if (sw == 0 || sh == 0 || dw == 0 || dh == 0) return fail(KB200_ERR_INVALID_ARGUMENT, "image dimensions must be non-zero");
    if (batch == 0) return fail(KB200_ERR_INVALID_ARGUMENT, "batch must be non-zero");
    return KB200_OK;
}
inline int check_ptr(const char* what, const void* p) {
    if (!p) return fail(KB200_ERR_INVALID_ARGUMENT, "null pointer for '%s'", what);
    return KB200_OK;
}

#define KB200_TRY(expr)                   \
    do {                                  \
        int _st = (expr);                 \
        if (_st != KB200_OK) return _st;  \
    } while (0)

struct DeviceInfo {
    int device = -1;
    int sm_count = 0;
    int cc_major = 0, cc_minor = 0;
    int max_smem_optin = 0;
};
const DeviceInfo& device_info();  // for the current device; cached, immutable after first use

inline cudaStream_t as_stream(kb200_stream_t s) { return reinterpret_cast<cudaStream_t>(s); }

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }
inline bool aligned4(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 3u) == 0; }

inline unsigned div_up(size_t a, size_t b) { return (unsigned)((a + b - 1) / b); }

// ── device helpers ──────────────────────────────────────────────────────────────────────────
#ifdef __CUDACC__

// 4:2:0 layouts (kb200_yuv420_layout): one tight w*h*3/2 buffer, Y plane first.  NV12 / NV21 interleave the chroma
// (U V / V U) at a w-byte row stride; I420 / YV12 store two (w/2 x h/2) planes, U then V / V then U.
static constexpr int YUV420_NV12 = KB200_YUV420_NV12, YUV420_NV21 = KB200_YUV420_NV21, YUV420_I420 = KB200_YUV420_I420,
                     YUV420_YV12 = KB200_YUV420_YV12;
__host__ __device__ constexpr bool yuv420_planar(int L) { return L == YUV420_I420 || L == YUV420_YV12; }
// byte offsets of the U and V planes of a planar frame (w, h even)
__host__ __device__ inline size_t yuv420_u_plane(int L, size_t w, size_t h) { return L == YUV420_I420 ? w * h : w * h + w * h / 4; }
__host__ __device__ inline size_t yuv420_v_plane(int L, size_t w, size_t h) { return L == YUV420_I420 ? w * h + w * h / 4 : w * h; }
// 4:4:4 as a layout beside the 4:2:0 ones, for the preprocess taps: three full-resolution planes Y, U, V (I444, I41x).
static constexpr int YUV444 = 4;

// 4:2:2 layouts (kb200_yuv422_layout): each 2-px group is one 32-bit word; Yuv422Bytes<L> gives the byte of Y0, Y1,
// U and V in it.  YUYV = Y0 U Y1 V, UYVY = U Y0 V Y1, YVYU = Y0 V Y1 U.
static constexpr int YUV422_YUYV = KB200_YUV422_YUYV, YUV422_UYVY = KB200_YUV422_UYVY, YUV422_YVYU = KB200_YUV422_YVYU;
template <int L> struct Yuv422Bytes { static constexpr int y0 = 0, y1 = 2, u = 1, v = 3; };
template <> struct Yuv422Bytes<YUV422_UYVY> { static constexpr int y0 = 1, y1 = 3, u = 0, v = 2; };
template <> struct Yuv422Bytes<YUV422_YVYU> { static constexpr int y0 = 0, y1 = 2, u = 3, v = 1; };

// Streaming (read-once / write-once) vector accesses: keep L1 for the gather taps.
__device__ __forceinline__ float4 ldg_stream_f4(const float4* p) {
    float4 v;
    asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p));
    return v;
}
__device__ __forceinline__ uint4 ldg_stream_u4(const uint4* p) {
    uint4 v;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
    return v;
}
__device__ __forceinline__ uint2 ldg_stream_u2(const uint2* p) {
    uint2 v;
    asm volatile("ld.global.nc.L1::no_allocate.v2.u32 {%0,%1}, [%2];" : "=r"(v.x), "=r"(v.y) : "l"(p));
    return v;
}
__device__ __forceinline__ void stg_stream_f4(float4* p, float4 v) {
    asm volatile("st.global.L1::no_allocate.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
__device__ __forceinline__ void stg_stream_u4(uint4* p, uint4 v) {
    asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ void stg_stream_f1(float* p, float v) {
    asm volatile("st.global.L1::no_allocate.f32 [%0], %1;" ::"l"(p), "f"(v) : "memory");
}

// Lane-wise fma.rn on two floats held as one 64-bit pair {lo, hi}.  sm_90 has no packed FP32 instruction, so each lane
// is one scalar FFMA; every lane rounds once, exactly like fmaf.  The pair form keeps the callers' register layout.
__device__ __forceinline__ unsigned long long fma2_rn(unsigned long long a, unsigned long long b, unsigned long long c) {
    float a0, a1, b0, b1, c0, c1, r0, r1;
    asm("mov.b64 {%0, %1}, %2;" : "=f"(a0), "=f"(a1) : "l"(a));
    asm("mov.b64 {%0, %1}, %2;" : "=f"(b0), "=f"(b1) : "l"(b));
    asm("mov.b64 {%0, %1}, %2;" : "=f"(c0), "=f"(c1) : "l"(c));
    asm("fma.rn.f32 %0, %1, %2, %3;" : "=f"(r0) : "f"(a0), "f"(b0), "f"(c0));
    asm("fma.rn.f32 %0, %1, %2, %3;" : "=f"(r1) : "f"(a1), "f"(b1), "f"(c1));
    unsigned long long r;
    asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(r0), "f"(r1));
    return r;
}

// byte `i` (0..3) of a 32-bit word -> exact float, through the 2^23 mantissa trick:
// PRMT builds 0x4B0000bb (= 8388608 + b) and one FADD removes the bias.  Exact for 0..255.
__device__ __forceinline__ float byte_to_float(uint32_t w, int i) {
    const uint32_t bits = __byte_perm(w, 0x4B000000u, 0x7650u + (uint32_t)i);  // {b_i, 0x00, 0x00, 0x4B}
    return __uint_as_float(bits) - 8388608.0f;
}

// Q20 YUV -> RGB decode, one coefficient set per kb200_yuv_matrix — color/yuv/kernels.rs:707-737 / preprocess.rs:501-508:
//   yy = max(Y - y_off, 0) * cy,  u = U - 128,  v = V - 128
//   R = sat((yy + cvr*v + 2^19) >> 20),  G = sat((yy + cug*u + cvg*v + 2^19) >> 20),  B = sat((yy + cub*u + 2^19) >> 20)
// The kernels take the set as a launch argument (the same kernels serve every matrix).  Every term is below 5.8e8 in
// magnitude, so the i32 sums cannot overflow.
struct YuvCoeffs {
    int y_off, cy, cvr, cub, cug, cvg;
};
// Indexed by kb200_yuv_matrix.  BT.601 limited keeps the reference's literal constants; the others are round(c * 2^20)
// of the exact coefficients from (Kr, Kb) = (0.299, 0.114) for BT.601 and (0.2126, 0.0722) for BT.709: cvr = 2(1-Kr),
// cub = 2(1-Kb), cug = -2Kb(1-Kb)/Kg, cvg = -2Kr(1-Kr)/Kg, with Kg = 1-Kr-Kb; limited range scales luma by 255/219
// and chroma by 255/224 (y_off 16), full range uses them as they are (y_off 0).
static constexpr YuvCoeffs YUV_COEFFS[4] = {
    {16, 1220542, 1673527, 2116026, -409993, -852492},   // KB200_YUV_BT601_LIMITED
    {0, 1048576, 1470104, 1858077, -360853, -748826},    // KB200_YUV_BT601_FULL
    {16, 1220945, 1879825, 2215014, -223607, -558796},   // KB200_YUV_BT709_LIMITED
    {0, 1048576, 1651297, 1945738, -196424, -490864},    // KB200_YUV_BT709_FULL
};
struct ChromaTerms {
    int b, g, r;  // cub*u + half, cug*u + cvg*v + half, cvr*v + half   (u, v already -128)
};
__device__ __forceinline__ ChromaTerms chroma_terms(int u, int v, const YuvCoeffs& c) {
    u -= 128;
    v -= 128;
    ChromaTerms t;
    t.b = c.cub * u + (1 << 19);
    t.g = c.cug * u + c.cvg * v + (1 << 19);
    t.r = c.cvr * v + (1 << 19);
    return t;
}
__device__ __forceinline__ int yy_term(int y, const YuvCoeffs& c) { return max(y - c.y_off, 0) * c.cy; }
__device__ __forceinline__ int sat_u8(int v) { return min(max(v, 0), 255); }
// integer adds are associative (two's complement, no overflow here: |terms| < 2^30), so
// (yy + CUB*u + half) == yy + (CUB*u + half) bit-for-bit.
__device__ __forceinline__ void decode_rgb(int yy, const ChromaTerms& t, int& r, int& g, int& b) {
    b = sat_u8((yy + t.b) >> 20);
    g = sat_u8((yy + t.g) >> 20);
    r = sat_u8((yy + t.r) >> 20);
}

// Q16 decode of n-bit codes (n = 10, 12: the 16-bit-word 4:2:0 formats P010, P012, I010, I012), the Q20 decode above
// rescaled.  With s = 2^(n-8) and W = 2^n - 1:
//   yy = max(Y - y_off, 0) * cy,  u = U - 128*s,  v = V - 128*s
//   R = clamp((yy + cvr*v + 2^15) >> 16, 0, W),  G = clamp((yy + cug*u + cvg*v + 2^15) >> 16, 0, W),  B = ... cub*u ...
// y_off = 16*s for limited range, 0 for full range.  The constants are round(c * 2^16) of the exact coefficients of the
// Q20 table's derivation, with the limited-range scales W/(219*s) for luma and W/(224*s) for chroma (1 for full range).
// At 12 bits every term is below 5.8e8 in magnitude, so the i32 sums cannot overflow.
// A 16-bit word holds its code in the high bits (P01x: code = word >> (16 - n)) or the low bits (I01x: word & W); the
// other bits are ignored, which also bounds every code by W.
static constexpr YuvCoeffs YUV16_COEFFS[2][4] = {   // [n == 12][kb200_yuv_matrix]
    {{64, 76533, 104905, 132590, -25750, -53435},    // 10 bits: KB200_YUV_BT601_LIMITED
     {0, 65536, 91881, 116130, -22553, -46802},      //          KB200_YUV_BT601_FULL
     {64, 76533, 117835, 138846, -14017, -35027},    //          KB200_YUV_BT709_LIMITED
     {0, 65536, 103206, 121609, -12276, -30679}},    //          KB200_YUV_BT709_FULL
    {{256, 76590, 104982, 132687, -25769, -53475},   // 12 bits
     {0, 65536, 91881, 116130, -22553, -46802},
     {256, 76590, 117921, 138947, -14027, -35053},
     {0, 65536, 103206, 121609, -12276, -30679}},
};
// One coefficient set of YUV16_COEFFS with the depth's code extraction: code = (word >> shift) & white.
struct Yuv16Coeffs {
    YuvCoeffs c;
    int shift;   // 16 - n for the MSB-aligned (P01x) layout, 0 for the LSB-aligned (I01x) one
    int white;   // W = 2^n - 1
};
inline Yuv16Coeffs yuv16_coeffs(int matrix, int bits, bool msb_aligned) {
    return {YUV16_COEFFS[bits == 12][matrix], msb_aligned ? 16 - bits : 0, (1 << bits) - 1};
}
__device__ __forceinline__ int yuv16_code(uint32_t word, const Yuv16Coeffs& k) { return (int)((word >> k.shift) & (uint32_t)k.white); }
__device__ __forceinline__ ChromaTerms chroma_terms16(int u, int v, const Yuv16Coeffs& k) {
    const int half = (k.white + 1) >> 1;   // 128 * s
    u -= half;
    v -= half;
    ChromaTerms t;
    t.b = k.c.cub * u + (1 << 15);
    t.g = k.c.cug * u + k.c.cvg * v + (1 << 15);
    t.r = k.c.cvr * v + (1 << 15);
    return t;
}
__device__ __forceinline__ int yy_term16(int y, const Yuv16Coeffs& k) { return max(y - k.c.y_off, 0) * k.c.cy; }
__device__ __forceinline__ void decode_rgb16(int yy, const ChromaTerms& t, int white, int& r, int& g, int& b) {
    b = min(max((yy + t.b) >> 16, 0), white);
    g = min(max((yy + t.g) >> 16, 0), white);
    r = min(max((yy + t.r) >> 16, 0), white);
}

#endif  // __CUDACC__

}  // namespace kb200
