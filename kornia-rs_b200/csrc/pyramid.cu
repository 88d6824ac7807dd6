// pyramid.cu — Gaussian pyramid levels: pyrdown / pyrup for f32 and u8 images (SURVEY §8(f) #4).
//
// Reference: pyramid.rs:22-250 (pyrup_f32, polyphase [1,4,6,4,1]/8 with the reference's own border rule), :252-427
// (reflect_101, pyrdown_f32: 25 taps, `sum += v * (ky*kx)` unfused, BORDER_REFLECT_101), :469-650 (pyrdown_u8: u16
// horizontal sums then (sum + 128) >> 8), :656-840 (pyrup_u8: (p + 6c + n + 4) >> 3 and (c + n + 1) >> 1 per pass with a
// u8 intermediate), GPU twins cuda/pyramid.rs.  The reference runs two passes through an intermediate buffer; every
// intermediate value is rounded to its storage type (f32 / u16 / u8) before the second pass, so computing it on the fly
// gives the same bits and the kernels below are single-pass: no scratch, one launch per level for the whole batch.
//
// Notes: these are small stencil kernels (each level is 1/4 of the previous one); a thread produces one destination
// pixel (pyrdown) or the 2x2 destination block of one source pixel (pyrup) for all channels; neighbouring threads share
// their taps through L1.  Batch = grid.z.
#include "kb200_common.cuh"

namespace kb200 {

__device__ __forceinline__ int reflect_101(int p, int len) {
    if (len == 1) return 0;
    if (p < 0) p = -p;
    const int period = 2 * (len - 1);
    p %= period;
    if (p >= len) p = period - p;
    return p;
}

// pyrdown_f32: dst(dx, dy) = sum over 5x5 of src(reflect(2dx + kx - 2), reflect(2dy + ky - 2)) * (k[ky] * k[kx]), ky outer
__global__ void __launch_bounds__(256) pyrdown_f32_kernel(const float* __restrict__ src, float* __restrict__ dst, uint32_t sw, uint32_t sh,
                                                          uint32_t dw, uint32_t dh, uint32_t C) {
    const uint32_t dx = blockIdx.x * 32u + threadIdx.x, dy = blockIdx.y * 8u + threadIdx.y;
    if (dx >= dw || dy >= dh) return;
    const float* s = src + (size_t)blockIdx.z * sw * sh * C;
    float* d = dst + ((size_t)blockIdx.z * dw * dh + (size_t)dy * dw + dx) * C;
    const float k1[5] = {0.0625f, 0.25f, 0.375f, 0.25f, 0.0625f};
    uint32_t xo[5];
#pragma unroll
    for (int t = 0; t < 5; ++t) xo[t] = (uint32_t)reflect_101((int)(dx * 2u) + t - 2, (int)sw) * C;
    float sum[4] = {0.0f, 0.0f, 0.0f, 0.0f};
#pragma unroll
    for (int ky = 0; ky < 5; ++ky) {
        const float* row = s + (size_t)reflect_101((int)(dy * 2u) + ky - 2, (int)sh) * sw * C;
#pragma unroll
        for (int kx = 0; kx < 5; ++kx) {
            const float w = k1[ky] * k1[kx];   // exact (powers of two times 1, 4, 6): the reference's precomputed table
            for (uint32_t c = 0; c < C; ++c) sum[c] += __ldg(row + xo[kx] + c) * w;
        }
    }
    for (uint32_t c = 0; c < C; ++c) d[c] = sum[c];
}

// horizontal pyrup value of one source row at even / odd destination column of source pixel x (pyramid.rs:22-90)
__device__ __forceinline__ void pyrup_h_f32(const float* __restrict__ row, uint32_t x, uint32_t sw, uint32_t C, uint32_t c, float* even, float* odd) {
    const float cur = __ldg(row + x * C + c);
    if (sw == 1u) { *even = cur; *odd = cur; return; }
    if (x == 0u) {
        const float r = __ldg(row + C + c);
        *even = (6.0f * cur + 2.0f * r) * 0.125f;
        *odd = (cur + r) * 0.5f;
    } else if (x == sw - 1u) {
        const float p = __ldg(row + (x - 1u) * C + c);
        *even = (1.0f * p + 7.0f * cur) * 0.125f;
        *odd = cur;
    } else {
        const float p = __ldg(row + (x - 1u) * C + c), n = __ldg(row + (x + 1u) * C + c);
        *even = (1.0f * p + 6.0f * cur + 1.0f * n) * 0.125f;
        *odd = (cur + n) * 0.5f;
    }
}

// one thread per source pixel: the 2x2 destination block (pyramid.rs:98-160 vertical rule on the horizontal values)
__global__ void __launch_bounds__(256) pyrup_f32_kernel(const float* __restrict__ src, float* __restrict__ dst, uint32_t sw, uint32_t sh, uint32_t C) {
    const uint32_t x = blockIdx.x * 32u + threadIdx.x, y = blockIdx.y * 8u + threadIdx.y;
    if (x >= sw || y >= sh) return;
    const float* s = src + (size_t)blockIdx.z * sw * sh * C;
    const uint32_t dw = sw * 2u;
    float* d = dst + ((size_t)blockIdx.z * dw * (sh * 2u) + (size_t)(2u * y) * dw + 2u * x) * C;
    uint32_t rt, rc, rb;
    if (sh == 1u) { rt = rc = rb = 0u; }
    else if (y == 0u) { rt = 0u; rc = 0u; rb = 1u; }
    else if (y == sh - 1u) { rt = sh - 2u; rc = sh - 1u; rb = sh - 1u; }
    else { rt = y - 1u; rc = y; rb = y + 1u; }
    const size_t rs = (size_t)sw * C;
    for (uint32_t c = 0; c < C; ++c) {
        float te, to, ce, co, be, bo;
        pyrup_h_f32(s + rt * rs, x, sw, C, c, &te, &to);
        pyrup_h_f32(s + rc * rs, x, sw, C, c, &ce, &co);
        pyrup_h_f32(s + rb * rs, x, sw, C, c, &be, &bo);
        float ee, eo, oe, oo;   // destination rows even / odd x columns even / odd
        if (y == 0u) {
            ee = (6.0f * ce + 2.0f * be) * 0.125f; eo = (6.0f * co + 2.0f * bo) * 0.125f;
            oe = (ce + be) * 0.5f; oo = (co + bo) * 0.5f;
        } else if (y == sh - 1u) {
            ee = (1.0f * te + 7.0f * ce) * 0.125f; eo = (1.0f * to + 7.0f * co) * 0.125f;
            oe = ce; oo = co;
        } else {
            ee = (1.0f * te + 6.0f * ce + 1.0f * be) * 0.125f; eo = (1.0f * to + 6.0f * co + 1.0f * bo) * 0.125f;
            oe = (ce + be) * 0.5f; oo = (co + bo) * 0.5f;
        }
        d[c] = ee; d[C + c] = eo;
        d[(size_t)dw * C + c] = oe; d[(size_t)dw * C + C + c] = oo;
    }
}

__global__ void __launch_bounds__(256) pyrdown_u8_kernel(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst, uint32_t sw, uint32_t sh,
                                                         uint32_t dw, uint32_t dh, uint32_t C) {
    const uint32_t dx = blockIdx.x * 32u + threadIdx.x, dy = blockIdx.y * 8u + threadIdx.y;
    if (dx >= dw || dy >= dh) return;
    const uint8_t* s = src + (size_t)blockIdx.z * sw * sh * C;
    uint8_t* d = dst + ((size_t)blockIdx.z * dw * dh + (size_t)dy * dw + dx) * C;
    uint32_t xo[5];
#pragma unroll
    for (int t = 0; t < 5; ++t) xo[t] = (uint32_t)reflect_101((int)(dx * 2u) + t - 2, (int)sw) * C;
    const uint32_t wv[5] = {1u, 4u, 6u, 4u, 1u};
    uint32_t acc[4] = {0u, 0u, 0u, 0u};
#pragma unroll
    for (int ky = 0; ky < 5; ++ky) {
        const uint8_t* row = s + (size_t)reflect_101((int)(dy * 2u) + ky - 2, (int)sh) * sw * C;
        for (uint32_t c = 0; c < C; ++c) {
            // u16 horizontal sum (<= 16 * 255), then the vertical weight — integer, exact in any order
            const uint32_t hsum = (uint32_t)row[xo[0] + c] + 4u * row[xo[1] + c] + 6u * row[xo[2] + c] + 4u * row[xo[3] + c] + row[xo[4] + c];
            acc[c] += wv[ky] * hsum;
        }
    }
    for (uint32_t c = 0; c < C; ++c) d[c] = (uint8_t)min((acc[c] + 128u) >> 8, 255u);
}

__device__ __forceinline__ void pyrup_h_u8(const uint8_t* __restrict__ row, uint32_t x, uint32_t sw, uint32_t C, uint32_t c, uint32_t* even, uint32_t* odd) {
    const uint32_t cur = row[x * C + c];
    const uint32_t p = row[(uint32_t)reflect_101((int)x - 1, (int)sw) * C + c], n = row[(uint32_t)reflect_101((int)x + 1, (int)sw) * C + c];
    *even = (p + 6u * cur + n + 4u) >> 3;
    *odd = (cur + n + 1u) >> 1;
}

__global__ void __launch_bounds__(256) pyrup_u8_kernel(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst, uint32_t sw, uint32_t sh, uint32_t C) {
    const uint32_t x = blockIdx.x * 32u + threadIdx.x, y = blockIdx.y * 8u + threadIdx.y;
    if (x >= sw || y >= sh) return;
    const uint8_t* s = src + (size_t)blockIdx.z * sw * sh * C;
    const uint32_t dw = sw * 2u;
    uint8_t* d = dst + ((size_t)blockIdx.z * dw * (sh * 2u) + (size_t)(2u * y) * dw + 2u * x) * C;
    const size_t rs = (size_t)sw * C;
    const uint8_t* rp = s + (size_t)reflect_101((int)y - 1, (int)sh) * rs;
    const uint8_t* rc = s + (size_t)y * rs;
    const uint8_t* rn = s + (size_t)reflect_101((int)y + 1, (int)sh) * rs;
    for (uint32_t c = 0; c < C; ++c) {
        uint32_t pe, po, ce, co, ne, no;
        pyrup_h_u8(rp, x, sw, C, c, &pe, &po);
        pyrup_h_u8(rc, x, sw, C, c, &ce, &co);
        pyrup_h_u8(rn, x, sw, C, c, &ne, &no);
        d[c] = (uint8_t)((pe + 6u * ce + ne + 4u) >> 3);
        d[C + c] = (uint8_t)((po + 6u * co + no + 4u) >> 3);
        d[(size_t)dw * C + c] = (uint8_t)((ce + ne + 1u) >> 1);
        d[(size_t)dw * C + C + c] = (uint8_t)((co + no + 1u) >> 1);
    }
}

template <typename T>
static int pyr_check(const T* src, size_t src_len, T* dst, size_t dst_len, uint32_t sw, uint32_t sh, uint32_t dw, uint32_t dh, uint32_t C,
                     uint32_t batch) {
    KB200_TRY(check_ptr("src", src)); KB200_TRY(check_ptr("dst", dst));
    KB200_TRY(check_geometry(sw, sh, dw, dh, batch));
    if (C == 0 || C > 4) return fail(KB200_ERR_UNSUPPORTED, "pyramid kernels support 1..4 channels, got %u", C);
    if (batch > 65535u) return fail(KB200_ERR_INVALID_ARGUMENT, "batch %u exceeds 65535 per call", batch);
    KB200_TRY(check_slice("src", src_len, (size_t)sw * sh * C * batch));
    KB200_TRY(check_slice("dst", dst_len, (size_t)dw * dh * C * batch));
    return KB200_OK;
}

}  // namespace kb200

using namespace kb200;

extern "C" {

KB200_API int kb200_pyrdown_f32(kb200_stream_t stream, const float* src, size_t src_len, float* dst, size_t dst_len, uint32_t sw, uint32_t sh,
                                uint32_t C, uint32_t batch) {
    const uint32_t dw = (sw + 1u) / 2u, dh = (sh + 1u) / 2u;
    KB200_TRY(pyr_check(src, src_len, dst, dst_len, sw, sh, dw, dh, C, batch));
    pyrdown_f32_kernel<<<dim3(div_up(dw, 32), div_up(dh, 8), batch), dim3(32, 8), 0, as_stream(stream)>>>(src, dst, sw, sh, dw, dh, C);
    return check_launch("pyrdown_f32_kernel");
}

KB200_API int kb200_pyrup_f32(kb200_stream_t stream, const float* src, size_t src_len, float* dst, size_t dst_len, uint32_t sw, uint32_t sh,
                              uint32_t C, uint32_t batch) {
    KB200_TRY(pyr_check(src, src_len, dst, dst_len, sw, sh, sw * 2u, sh * 2u, C, batch));
    pyrup_f32_kernel<<<dim3(div_up(sw, 32), div_up(sh, 8), batch), dim3(32, 8), 0, as_stream(stream)>>>(src, dst, sw, sh, C);
    return check_launch("pyrup_f32_kernel");
}

KB200_API int kb200_pyrdown_u8(kb200_stream_t stream, const uint8_t* src, size_t src_len, uint8_t* dst, size_t dst_len, uint32_t sw, uint32_t sh,
                               uint32_t C, uint32_t batch) {
    const uint32_t dw = (sw + 1u) / 2u, dh = (sh + 1u) / 2u;
    KB200_TRY(pyr_check(src, src_len, dst, dst_len, sw, sh, dw, dh, C, batch));
    pyrdown_u8_kernel<<<dim3(div_up(dw, 32), div_up(dh, 8), batch), dim3(32, 8), 0, as_stream(stream)>>>(src, dst, sw, sh, dw, dh, C);
    return check_launch("pyrdown_u8_kernel");
}

KB200_API int kb200_pyrup_u8(kb200_stream_t stream, const uint8_t* src, size_t src_len, uint8_t* dst, size_t dst_len, uint32_t sw, uint32_t sh,
                             uint32_t C, uint32_t batch) {
    KB200_TRY(pyr_check(src, src_len, dst, dst_len, sw, sh, sw * 2u, sh * 2u, C, batch));
    pyrup_u8_kernel<<<dim3(div_up(sw, 32), div_up(sh, 8), batch), dim3(32, 8), 0, as_stream(stream)>>>(src, dst, sw, sh, C);
    return check_launch("pyrup_u8_kernel");
}

}  // extern "C"
