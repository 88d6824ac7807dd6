// u8_sampler.cuh — the Q10 bilinear blend of the u8 warps / remap (warp/common.rs:14-181) with WORD-granular taps.
//
// The byte version issues 12 `LDG.U8` per RGB pixel (4 taps x 3 channels); ncu on the round-1 kernels showed them bound
// by LSU instructions, far from DRAM.  The two taps of a row are six consecutive bytes, so
// three aligned 32-bit words per row cover them: 6 `LDG.32` + two funnel shifts per row instead of 12 byte loads.  The
// arithmetic is unchanged — `(top*fy1 + bot*fy + 2^19) >> 20` with `top = p0*fx1 + p1*fx` — and bit-exact.
#pragma once

#include <stdint.h>

namespace kb200 {

// `img` is 4-byte aligned, `img_bytes` = sw*sh*3.  Taps (xi, yi), (xi1, yi), (xi, yi1), (xi1, yi1) with xi1 in {xi, xi+1}.
// Returns false (nothing written) when the 12-byte window of a row would run past the image — the caller's byte path
// handles those few pixels at the very end of the image.
__device__ __forceinline__ bool q10_blend_c3_words(const uint8_t* __restrict__ img, uint32_t img_bytes, int sw, int xi, int yi, int xi1, int yi1,
                                                   uint32_t fx, uint32_t fy, uint8_t* __restrict__ d) {
    const uint32_t o0 = ((uint32_t)yi * (uint32_t)sw + (uint32_t)xi) * 3u, o1 = ((uint32_t)yi1 * (uint32_t)sw + (uint32_t)xi) * 3u;
    const uint32_t b0 = o0 & ~3u, b1 = o1 & ~3u;
    if (max(b0, b1) + 12u > img_bytes) return false;
    const uint32_t* w0 = reinterpret_cast<const uint32_t*>(img + b0);
    const uint32_t* w1 = reinterpret_cast<const uint32_t*>(img + b1);
    const uint32_t a0 = __ldg(w0), a1 = __ldg(w0 + 1), a2 = __ldg(w0 + 2);
    const uint32_t c0 = __ldg(w1), c1 = __ldg(w1 + 1), c2 = __ldg(w1 + 2);
    const uint32_t s0 = (o0 & 3u) * 8u, s1 = (o1 & 3u) * 8u;
    const uint32_t lo0 = __funnelshift_r(a0, a1, s0), hi0 = __funnelshift_r(a1, a2, s0);   // bytes o..o+3 | o+4..o+7
    const uint32_t lo1 = __funnelshift_r(c0, c1, s1), hi1 = __funnelshift_r(c1, c2, s1);
    const bool dup = xi1 == xi;            // right edge: the +1 tap is the pixel itself
    const uint32_t fx1 = 1024u - fx, fy1 = 1024u - fy;
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
        const uint32_t p00 = (lo0 >> (8 * ch)) & 0xFFu, p10 = (lo1 >> (8 * ch)) & 0xFFu;
        const uint32_t n0 = ch == 0 ? (lo0 >> 24) : ((hi0 >> (8 * (ch - 1))) & 0xFFu);
        const uint32_t n1 = ch == 0 ? (lo1 >> 24) : ((hi1 >> (8 * (ch - 1))) & 0xFFu);
        const uint32_t p01 = dup ? p00 : n0, p11 = dup ? p10 : n1;
        const uint32_t top = p00 * fx1 + p01 * fx;
        const uint32_t bot = p10 * fx1 + p11 * fx;
        d[ch] = (uint8_t)((top * fy1 + bot * fy + (1u << 19)) >> 20);
    }
    return true;
}

// Interior form (round 2, second pass).  ncu on the u8 warps: issue-bound — the
// clamps, the +1-tap selects, the window test and the two-stage blend run for every pixel although only the image border
// needs them.  For a pixel whose taps (xi, yi) .. (xi+1, yi+1) are all inside and yi + 2 < sh (so both 12-byte windows stay
// inside the image: the callers' fast predicate), the sampler is: 6 LDG.32, 4 funnel shifts (the shifter uses the low five
// bits of o*8), four 2-D weights, and per channel 4 byte extractions + 4 IMAD + 1 shift.
//   (top*fy1 + bot*fy + 2^19) >> 20 with top = p00*fx1 + p01*fx, bot = p10*fx1 + p11*fx
//     == (p00*fx1*fy1 + p01*fx*fy1 + p10*fx1*fy + p11*fx*fy + 2^19) >> 20   — integer arithmetic, every term < 2^28.
// `img` is 4-byte aligned, row3 = sw * 3.
__device__ __forceinline__ void q10_blend_c3_interior(const uint8_t* __restrict__ img, uint32_t row3, uint32_t xi, uint32_t yi, uint32_t fx, uint32_t fy,
                                                      uint32_t* r0, uint32_t* r1, uint32_t* r2) {
    const uint32_t o0 = yi * row3 + xi * 3u, o1 = o0 + row3;
    const uint32_t* w0 = reinterpret_cast<const uint32_t*>(img + (o0 & ~3u));
    const uint32_t* w1 = reinterpret_cast<const uint32_t*>(img + (o1 & ~3u));
    const uint32_t a0 = __ldg(w0), a1 = __ldg(w0 + 1), a2 = __ldg(w0 + 2);
    const uint32_t c0 = __ldg(w1), c1 = __ldg(w1 + 1), c2 = __ldg(w1 + 2);
    const uint32_t s0 = o0 * 8u, s1 = o1 * 8u;
    const uint32_t lo0 = __funnelshift_r(a0, a1, s0), hi0 = __funnelshift_r(a1, a2, s0);   // bytes o..o+3 | o+4..o+7
    const uint32_t lo1 = __funnelshift_r(c0, c1, s1), hi1 = __funnelshift_r(c1, c2, s1);
    const uint32_t fx1 = 1024u - fx, fy1 = 1024u - fy;
    const uint32_t W00 = fx1 * fy1, W01 = fx * fy1, W10 = fx1 * fy, W11 = fx * fy;
    uint32_t r[3];
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
        const uint32_t p00 = __byte_perm(lo0, 0u, 0x4440u + ch), p10 = __byte_perm(lo1, 0u, 0x4440u + ch);
        const uint32_t p01 = ch == 0 ? (lo0 >> 24) : __byte_perm(hi0, 0u, 0x4440u + (ch - 1));
        const uint32_t p11 = ch == 0 ? (lo1 >> 24) : __byte_perm(hi1, 0u, 0x4440u + (ch - 1));
        r[ch] = (p00 * W00 + p01 * W01 + p10 * W10 + p11 * W11 + (1u << 19)) >> 20;
    }
    *r0 = r[0]; *r1 = r[1]; *r2 = r[2];
}

}  // namespace kb200
