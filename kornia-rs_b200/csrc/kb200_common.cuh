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
    KNOB_FR_NPX = 0, KNOB_FR_STAGES, KNOB_FR_CTAS,          // fused_rows (resize_fused.cu)
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

// BT.601 limited-range Q20 decode — color/yuv/kernels.rs:707-737 / preprocess.rs:501-508.
struct ChromaTerms {
    int b, g, r;  // CUB*u + half, CUG*u + CVG*v + half, CVR*v + half   (u, v already -128)
};
__device__ __forceinline__ ChromaTerms chroma_terms(int u, int v) {
    u -= 128;
    v -= 128;
    ChromaTerms t;
    t.b = 2116026 * u + (1 << 19);
    t.g = (-409993) * u + (-852492) * v + (1 << 19);
    t.r = 1673527 * v + (1 << 19);
    return t;
}
__device__ __forceinline__ int yy_term(int y) { return max(y - 16, 0) * 1220542; }
__device__ __forceinline__ int sat_u8(int v) { return min(max(v, 0), 255); }
// integer adds are associative (two's complement, no overflow here: |terms| < 2^30), so
// (yy + CUB*u + half) == yy + (CUB*u + half) bit-for-bit.
__device__ __forceinline__ void decode_rgb(int yy, const ChromaTerms& t, int& r, int& g, int& b) {
    b = sat_u8((yy + t.b) >> 20);
    g = sat_u8((yy + t.g) >> 20);
    r = sat_u8((yy + t.r) >> 20);
}

#endif  // __CUDACC__

}  // namespace kb200
