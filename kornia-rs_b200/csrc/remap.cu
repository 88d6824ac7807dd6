// remap.cu — generic geometric transformation by coordinate maps (SURVEY §8(f) #2).
//
// Reference: interpolation/remap.rs:43-128 (f32: bilinear_interpolation / nearest_neighbor_interpolation per pixel at
// (map_x, map_y)), :157-296 (u8: Q10 sampler of the u8 warps, nearest with constant-0 border); device twins
// cuda/remap.rs:61-158, :381-470.  Coordinates outside [0,w) x [0,h) — NaN included — produce 0.
// The maps are shared by every image of a batch (one undistortion map, many frames).
//
// Per pixel: 8 B of map + the taps + the output; taps of neighbouring pixels overlap for smooth maps, so L1 serves
// most of them.  Thread per destination pixel, map reads lane-contiguous.
#include "kb200_common.cuh"
#include "u8_sampler.cuh"

namespace kb200 {

// interpolation/bilinear.rs:16-66 for an in-range (u, v): val00-replicate rule, weights formed first, left-to-right sum
__device__ __forceinline__ void remap_bilinear_f32_c3(const float* __restrict__ s, uint32_t sw, uint32_t sh, float u, float v, float* __restrict__ d) {
    const uint32_t iu = (uint32_t)u, iv = (uint32_t)v;   // trunc; u, v >= 0
    const float fu = u - truncf(u), fv = v - truncf(v);
    const bool hx = iu + 1u < sw, hy = iv + 1u < sh;
    const uint32_t row = sw * 3u;
    const uint32_t o00 = iv * row + iu * 3u;
    const uint32_t o01 = hx ? o00 + 3u : o00, o10 = hy ? o00 + row : o00, o11 = (hx && hy) ? o00 + row + 3u : o00;
    const float fuu = 1.0f - fu, fvv = 1.0f - fv;
    const float w00 = fvv * fuu, w10 = fvv * fu, w01 = fv * fuu, w11 = fv * fu;
#pragma unroll
    for (int c = 0; c < 3; ++c) d[c] = w00 * __ldg(s + o00 + c) + w10 * __ldg(s + o01 + c) + w01 * __ldg(s + o10 + c) + w11 * __ldg(s + o11 + c);
}

template <bool BILINEAR>
__global__ void __launch_bounds__(256) remap_f32_c3_kernel(const float* __restrict__ src, float* __restrict__ dst, const float* __restrict__ map_x,
                                                           const float* __restrict__ map_y, uint32_t sw, uint32_t sh, uint32_t npx) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= npx) return;
    const float* s = src + (size_t)blockIdx.y * sw * sh * 3;
    float* d = dst + ((size_t)blockIdx.y * npx + i) * 3;
    const float x = __ldg(map_x + i), y = __ldg(map_y + i);
    if (!(x >= 0.0f && x < (float)sw && y >= 0.0f && y < (float)sh)) { d[0] = 0.0f; d[1] = 0.0f; d[2] = 0.0f; return; }
    if (BILINEAR) { remap_bilinear_f32_c3(s, sw, sh, x, y, d); return; }
    const uint32_t xi = min((uint32_t)roundf(x), sw - 1u), yi = min((uint32_t)roundf(y), sh - 1u);   // interpolation/nearest.rs:15-30
    const float* p = s + ((size_t)yi * sw + xi) * 3;
    d[0] = __ldg(p); d[1] = __ldg(p + 1); d[2] = __ldg(p + 2);
}

template <int C, bool BILINEAR>
__device__ __forceinline__ void remap_u8_general_pixel(const uint8_t* __restrict__ s, uint8_t* __restrict__ d, float xf, float yf, int sw, int sh, bool words);

constexpr uint32_t REMAP_U8_PX = 4;      // pixels per thread (i, i + 256, ...): the per-thread set-up is a third of a one-pixel thread

template <int C, bool BILINEAR>
__global__ void __launch_bounds__(256) remap_u8_kernel(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst, const float* __restrict__ map_x,
                                                       const float* __restrict__ map_y, int sw, int sh, uint32_t npx, bool words, bool aligned,
                                                       bool img_fast) {
    // image fastest when the grid allows: the maps (8 of the 14 bytes a pixel moves) are shared by the batch — consecutive
    // blocks then work on the same map span for different images and find it in L2 instead of re-reading it per image
    const uint32_t img = img_fast ? blockIdx.x : blockIdx.y, blk = img_fast ? blockIdx.y : blockIdx.x;
    const uint8_t* s = src + (size_t)img * sw * sh * C;
    uint8_t* dimg = dst + (size_t)img * npx * C;
    const bool fast_ok = BILINEAR && C == 3 && aligned && sw >= 4 && sh >= 3;
    const float xlim = (float)(sw - 1), ylim = (float)(sh - 2);
#pragma unroll
    for (uint32_t j = 0; j < REMAP_U8_PX; ++j) {
        const uint32_t ir = (blk * REMAP_U8_PX + j) * 256u + threadIdx.x;
        if ((ir & ~31u) >= npx) return;                     // whole warp
        const bool live = ir < npx;
        const uint32_t i = live ? ir : npx - 1u;            // lanes past the end recompute the last pixel and store nothing
        uint8_t* d = dimg + (size_t)i * C;
        const float xf = __ldg(map_x + i), yf = __ldg(map_y + i);
        // interior fast path (u8_sampler.cuh): in range (NaN / inf fail), all taps inside, two rows of slack below
        const bool fastpix = fast_ok && xf >= 0.0f && xf < xlim && yf >= 0.0f && yf < ylim;
        if (__all_sync(0xFFFFFFFFu, fastpix)) {
            const uint32_t xi = (uint32_t)xf, yi = (uint32_t)yf;          // floor == trunc here
            const uint32_t fx = __float2uint_rz((xf - (float)xi) * 1024.0f), fy = __float2uint_rz((yf - (float)yi) * 1024.0f);
            uint32_t r0, r1, r2;
            q10_blend_c3_interior(s, (uint32_t)sw * 3u, xi, yi, fx, fy, &r0, &r1, &r2);
            if (live) { d[0] = (uint8_t)r0; d[1] = (uint8_t)r1; d[2] = (uint8_t)r2; }
            continue;
        }
        if (live) remap_u8_general_pixel<C, BILINEAR>(s, d, xf, yf, sw, sh, words);
    }
}

template <int C, bool BILINEAR>
__device__ __forceinline__ void remap_u8_general_pixel(const uint8_t* __restrict__ s, uint8_t* __restrict__ d, float xf, float yf, int sw, int sh, bool words) {
    bool ok;
    if (BILINEAR) ok = isfinite(xf) && isfinite(yf);
    else ok = xf >= 0.0f && xf < (float)sw && yf >= 0.0f && yf < (float)sh;
    int xi = 0, yi = 0;
    if (ok && BILINEAR) {   // remap.rs:249-264
        xi = __float2int_rz(floorf(xf)); yi = __float2int_rz(floorf(yf));
        ok = xi >= 0 && xi < sw && yi >= 0 && yi < sh;
    }
    if (!ok) {
#pragma unroll
        for (int ch = 0; ch < C; ++ch) d[ch] = 0;
        return;
    }
    if (!BILINEAR) {        // remap.rs:283-291
        xi = min(max(__float2int_rz(roundf(xf)), 0), sw - 1); yi = min(max(__float2int_rz(roundf(yf)), 0), sh - 1);
        const uint8_t* p = s + ((size_t)yi * sw + xi) * C;
#pragma unroll
        for (int ch = 0; ch < C; ++ch) d[ch] = p[ch];
        return;
    }
    // Q10 blend, warp/common.rs:80-181 (scalar form)
    const uint32_t fx = __float2uint_rz((xf - (float)xi) * 1024.0f), fy = __float2uint_rz((yf - (float)yi) * 1024.0f);
    const uint32_t fx1 = 1024u - fx, fy1 = 1024u - fy;
    const int xi1 = (xi + 1 < sw) ? xi + 1 : xi, yi1 = (yi + 1 < sh) ? yi + 1 : yi;
    if (C == 3 && words && q10_blend_c3_words(s, (uint32_t)sw * (uint32_t)sh * 3u, sw, xi, yi, xi1, yi1, fx, fy, d)) return;
    const uint8_t* r0 = s + (size_t)yi * sw * C;
    const uint8_t* r1 = s + (size_t)yi1 * sw * C;
#pragma unroll
    for (int ch = 0; ch < C; ++ch) {
        const uint32_t top = r0[xi * C + ch] * fx1 + r0[xi1 * C + ch] * fx;
        const uint32_t bot = r1[xi * C + ch] * fx1 + r1[xi1 * C + ch] * fx;
        d[ch] = (uint8_t)((top * fy1 + bot * fy + (1u << 19)) >> 20);
    }
}

static int remap_check(const void* src, const void* dst, const void* mx, const void* my, uint32_t sw, uint32_t sh, uint32_t dw, uint32_t dh,
                       uint32_t batch, size_t map_len, int interp) {
    KB200_TRY(check_ptr("src", src)); KB200_TRY(check_ptr("dst", dst)); KB200_TRY(check_ptr("map_x", mx)); KB200_TRY(check_ptr("map_y", my));
    KB200_TRY(check_geometry(sw, sh, dw, dh, batch));
    if (batch > 65535u) return fail(KB200_ERR_INVALID_ARGUMENT, "batch %u exceeds 65535 per call", batch);
    if (interp != KB200_INTERP_NEAREST && interp != KB200_INTERP_BILINEAR)
        return fail(KB200_ERR_UNSUPPORTED, "CUDA remap supports Nearest/Bilinear only (mode %d)", interp);
    if ((size_t)dw * dh > 0xFFFFFFFFull || (size_t)sw * sh * 4 > 0xFFFFFFFFull) return fail(KB200_ERR_DIMS_TOO_LARGE, "remap image dimensions too large");
    KB200_TRY(check_slice("map", map_len, (size_t)dw * dh));
    return KB200_OK;
}

bool launch_remap_lean(cudaStream_t s, const float* src, float* dst, const float* map_x, const float* map_y, uint32_t sw, uint32_t sh, uint32_t dw,
                       uint32_t dh, uint32_t batch, int* status);   // warp.cu

}  // namespace kb200

using namespace kb200;

extern "C" {

KB200_API int kb200_remap_f32_c3(kb200_stream_t stream, const float* src, size_t src_len, float* dst, size_t dst_len, const float* map_x,
                                 const float* map_y, size_t map_len, uint32_t sw, uint32_t sh, uint32_t dw, uint32_t dh, uint32_t batch,
                                 int interp) {
    KB200_TRY(remap_check(src, dst, map_x, map_y, sw, sh, dw, dh, batch, map_len, interp));
    KB200_TRY(check_slice("src", src_len, (size_t)sw * sh * 3 * batch));
    KB200_TRY(check_slice("dst", dst_len, (size_t)dw * dh * 3 * batch));
    const uint32_t npx = dw * dh;
    dim3 grid(div_up(npx, 256u), batch);
    cudaStream_t s = as_stream(stream);
    if (interp == KB200_INTERP_BILINEAR) {
        // round 2: the lean bilinear gather of the warps, coordinates from the maps (warp.cu) — four rows per thread, interior
        // fast path, TMA tile stores
        int st = KB200_OK;
        if (launch_remap_lean(s, src, dst, map_x, map_y, sw, sh, dw, dh, batch, &st)) return st;
    }
    if (interp == KB200_INTERP_BILINEAR) remap_f32_c3_kernel<true><<<grid, 256, 0, s>>>(src, dst, map_x, map_y, sw, sh, npx);
    else remap_f32_c3_kernel<false><<<grid, 256, 0, s>>>(src, dst, map_x, map_y, sw, sh, npx);
    return check_launch("remap_f32_c3_kernel");
}

KB200_API int kb200_remap_u8(kb200_stream_t stream, const uint8_t* src, size_t src_len, uint8_t* dst, size_t dst_len, const float* map_x,
                             const float* map_y, size_t map_len, uint32_t sw, uint32_t sh, uint32_t dw, uint32_t dh, uint32_t channels,
                             uint32_t batch, int interp) {
    KB200_TRY(remap_check(src, dst, map_x, map_y, sw, sh, dw, dh, batch, map_len, interp));
    const uint32_t C = channels;
    if (!(C == 1 || C == 3 || C == 4)) return fail(KB200_ERR_UNSUPPORTED, "u8 remap supports 1, 3 or 4 channels, got %u", C);
    KB200_TRY(check_slice("src", src_len, (size_t)sw * sh * C * batch));
    KB200_TRY(check_slice("dst", dst_len, (size_t)dw * dh * C * batch));
    const uint32_t npx = dw * dh;
    const uint32_t nblk = div_up(npx, 256u * REMAP_U8_PX);
    const bool img_fast = nblk <= 65535u;
    dim3 grid(img_fast ? batch : nblk, img_fast ? nblk : batch);
    cudaStream_t s = as_stream(stream);
    const bool bil = interp == KB200_INTERP_BILINEAR;
    // word taps measured neutral-to-slower for remap: off unless knob b = 2
    const bool aligned = C == 3 && knob(KNOB_B) != 1 && (reinterpret_cast<uintptr_t>(src) & 3u) == 0 && (batch == 1 || ((size_t)sw * sh * 3) % 4 == 0);
    const bool words = aligned && knob(KNOB_B) == 2;
#define KB200_REMAP_U8(CC)                                                                                         \
    if (C == CC) {                                                                                                 \
        if (bil) remap_u8_kernel<CC, true><<<grid, 256, 0, s>>>(src, dst, map_x, map_y, (int)sw, (int)sh, npx, words, aligned, img_fast);     \
        else remap_u8_kernel<CC, false><<<grid, 256, 0, s>>>(src, dst, map_x, map_y, (int)sw, (int)sh, npx, words, aligned, img_fast);        \
    }
    KB200_REMAP_U8(1) KB200_REMAP_U8(3) KB200_REMAP_U8(4)
#undef KB200_REMAP_U8
    return check_launch("remap_u8_kernel");
}

}  // extern "C"
