// resample_hq.cu — bicubic (Keys a = -0.5) and Lanczos-3 samplers for resize and the warps (SURVEY §8(f) #3).
//
// Reference: interpolation/bicubic.rs:12-61, interpolation/lanczos.rs:16-236 (CPU), GPU twins cuda/resize.rs:244-402,
// cuda/warp_affine.rs:224-448, cuda/warp_perspective.rs:174-381.  The reference keeps CPU and GPU byte-exact here by
// writing `mul_add` / `fmaf` explicitly where a step is fused and plain mul/add (unfused under --fmad=false) elsewhere;
// this file follows the same split (it is compiled with -fmad=false like the rest of the library):
//   Keys weights   Horner chains of fmaf (bicubic.rs:17-26)
//   bicubic        w = wx*wy (plain), acc = fmaf(w, v, acc), dy outer / dx inner (bicubic.rs:48-58)
//   sin(pi x)      integer reduction + odd Taylor polynomial in plain mul/add (lanczos.rs:19-35) — no libm sin
//   Lanczos warp   six weights from four sin_pi, per-axis normalisation (sum left to right, one reciprocal, six
//                  multiplies), rx = fmaf(wx, v, rx) per row, acc = fmaf(wy, rx, acc) (lanczos.rs:106-181)
//   Lanczos resize separable: per-axis tables (tap base + six normalised weights per destination index, lanczos.rs:59-92),
//                  H pass into an f32 intermediate of dst_w x src_h, then V pass, both fmaf chains (lanczos.rs:187-236).
//
// Notes.  These are the reference's "quality" samplers: 16 / 36 taps per pixel, compute-heavier and rarely on a
// camera pipeline's critical path.  Thread per destination pixel with batch = grid.z; the tables of the separable
// Lanczos resize are built ON THE DEVICE by a small table kernel with the host code's own expression trees (same IEEE
// operations -> same bits as the reference's host-built tables), into the caller's scratch buffer — nothing is
// allocated or uploaded, so the launch stays asynchronous and graph-capturable (the reference allocates and uploads
// inside launch_resize_lanczos_cuda, cuda/resize.rs:868-884).
#include "kb200_common.cuh"

namespace kb200 {

struct HqMat { float m[9]; };

__device__ __forceinline__ void keys_weights(float frac, float w[4]) {
    float t;
    t = 1.0f + frac; w[0] = fmaf(fmaf(fmaf(-0.5f, t, 2.5f), t, -4.0f), t, 2.0f);
    t = frac;        w[1] = fmaf(fmaf(1.5f, t, -2.5f) * t, t, 1.0f);
    t = 1.0f - frac; w[2] = fmaf(fmaf(1.5f, t, -2.5f) * t, t, 1.0f);
    t = 2.0f - frac; w[3] = fmaf(fmaf(fmaf(-0.5f, t, 2.5f), t, -4.0f), t, 2.0f);
}

__device__ __forceinline__ float hq_sin_pi(float x) {
    const float k = roundf(x);
    const float r = x - k;
    const float z = 3.14159265358979323846f * r;
    const float z2 = z * z;
    float p = -2.5052108e-8f;
    p = p * z2 + 2.7557319e-6f;
    p = p * z2 + -1.984127e-4f;
    p = p * z2 + 8.333334e-3f;
    p = p * z2 + -1.6666667e-1f;
    const float s = z + z * z2 * p;
    return (((int)k) & 1) ? -s : s;
}

__device__ __forceinline__ float hq_lanczos3(float x) {
    if (fabsf(x) < 1e-5f) return 1.0f;
    if (fabsf(x) >= 3.0f) return 0.0f;
    const float pix = 3.14159265358979323846f * x;
    const float pix3 = pix * 0.33333334f;
    return __fdiv_rn(hq_sin_pi(x) * hq_sin_pi(x * (1.0f / 3.0f)), pix * pix3);
}

__device__ __forceinline__ float hq_den(float x) {
    const float pix = 3.14159265358979323846f * x;
    const float pix3 = pix * 0.33333334f;
    return pix * pix3;
}

// six normalised weights of the warp samplers (lanczos.rs:106-137 + :158-167)
__device__ __forceinline__ void lanczos3_weights_norm(float frac, float w[6]) {
    const float s = hq_sin_pi(frac);
    const float t0 = hq_sin_pi(frac * (1.0f / 3.0f));
    const float t1 = hq_sin_pi((frac - 1.0f) * (1.0f / 3.0f));
    const float t2 = hq_sin_pi((frac - 2.0f) * (1.0f / 3.0f));
    const float st0 = s * t0, st1 = s * t1, st2 = s * t2;
    w[0] = __fdiv_rn(-st1, hq_den(frac + 2.0f));
    w[1] = __fdiv_rn(st2, hq_den(frac + 1.0f));
    w[2] = __fdiv_rn(st0, hq_den(frac));
    w[3] = __fdiv_rn(-st1, hq_den(frac - 1.0f));
    w[4] = __fdiv_rn(st2, hq_den(frac - 2.0f));
    w[5] = __fdiv_rn(st0, hq_den(frac - 3.0f));
    if (frac < 1e-5f) w[2] = 1.0f;
    if (fabsf(frac - 1.0f) < 1e-5f) w[3] = 1.0f;
    const float sum = w[0] + w[1] + w[2] + w[3] + w[4] + w[5];
    const float inv = __fdiv_rn(1.0f, sum);
#pragma unroll
    for (int i = 0; i < 6; ++i) w[i] *= inv;
}

// 4x4 bicubic sample of all three channels at (sx, sy); taps replicate-clamped per axis
__device__ __forceinline__ void sample_bicubic_c3(const float* __restrict__ s, uint32_t sw, uint32_t sh, float sx, float sy, float out[3]) {
    const float x0f = floorf(sx), y0f = floorf(sy);
    float wx[4], wy[4];
    keys_weights(sx - x0f, wx);
    keys_weights(sy - y0f, wy);
    const int x0 = (int)x0f, y0 = (int)y0f;
    uint32_t xo[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) xo[i] = (uint32_t)max(0, min(x0 + i - 1, (int)sw - 1)) * 3u;
    float a0 = 0.0f, a1 = 0.0f, a2 = 0.0f;
#pragma unroll
    for (int dy = 0; dy < 4; ++dy) {
        const float* row = s + (size_t)max(0, min(y0 + dy - 1, (int)sh - 1)) * sw * 3u;
#pragma unroll
        for (int dx = 0; dx < 4; ++dx) {
            const float w = wx[dx] * wy[dy];
            const float* p = row + xo[dx];
            a0 = fmaf(w, __ldg(p), a0);
            a1 = fmaf(w, __ldg(p + 1), a1);
            a2 = fmaf(w, __ldg(p + 2), a2);
        }
    }
    out[0] = a0; out[1] = a1; out[2] = a2;
}

// 6x6 Lanczos-3 sample: per-row fmaf over dx, then fmaf of the row result by wy[dy]
__device__ __forceinline__ void sample_lanczos_c3(const float* __restrict__ s, uint32_t sw, uint32_t sh, float sx, float sy, float out[3]) {
    const float x0f = floorf(sx), y0f = floorf(sy);
    float wx[6], wy[6];
    lanczos3_weights_norm(sx - x0f, wx);
    lanczos3_weights_norm(sy - y0f, wy);
    const int x0 = (int)x0f, y0 = (int)y0f;
    uint32_t xo[6];
#pragma unroll
    for (int i = 0; i < 6; ++i) xo[i] = (uint32_t)max(0, min(x0 + i - 2, (int)sw - 1)) * 3u;
    float a0 = 0.0f, a1 = 0.0f, a2 = 0.0f;
#pragma unroll
    for (int dy = 0; dy < 6; ++dy) {
        const float* row = s + (size_t)max(0, min(y0 + dy - 2, (int)sh - 1)) * sw * 3u;
        float r0 = 0.0f, r1 = 0.0f, r2 = 0.0f;
#pragma unroll
        for (int dx = 0; dx < 6; ++dx) {
            const float* p = row + xo[dx];
            r0 = fmaf(wx[dx], __ldg(p), r0);
            r1 = fmaf(wx[dx], __ldg(p + 1), r1);
            r2 = fmaf(wx[dx], __ldg(p + 2), r2);
        }
        a0 = fmaf(wy[dy], r0, a0);
        a1 = fmaf(wy[dy], r1, a1);
        a2 = fmaf(wy[dy], r2, a2);
    }
    out[0] = a0; out[1] = a1; out[2] = a2;
}

// ── resize ───────────────────────────────────────────────────────────────────────────────────
// cuda/resize.rs:245-308: coordinate a*x + b (unfused), clamped to [0, len-1]
__global__ void __launch_bounds__(256) resize_bicubic_c3_kernel(const float* __restrict__ src, float* __restrict__ dst, uint32_t sw, uint32_t sh,
                                                                uint32_t dw, uint32_t dh, float ax, float bx, float ay, float by) {
    const uint32_t x = blockIdx.x * 32u + threadIdx.x, y = blockIdx.y * 8u + threadIdx.y;
    if (x >= dw || y >= dh) return;
    const float* s = src + (size_t)blockIdx.z * sw * sh * 3u;
    float* d = dst + ((size_t)blockIdx.z * dw * dh + (size_t)y * dw + x) * 3u;
    const float sx = fmaxf(fminf(ax * (float)x + bx, (float)(sw - 1u)), 0.0f);
    const float sy = fmaxf(fminf(ay * (float)y + by, (float)(sh - 1u)), 0.0f);
    float v[3];
    sample_bicubic_c3(s, sw, sh, sx, sy, v);
    d[0] = v[0]; d[1] = v[1]; d[2] = v[2];
}

// lanczos_axis (lanczos.rs:59-92) on the device: one thread per destination index of one axis
__global__ void lanczos_axis_kernel(uint32_t src_len, uint32_t dst_len, int* __restrict__ x0s, float* __restrict__ wtab) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= dst_len) return;
    const float a = __fdiv_rn((float)src_len, (float)dst_len);
    const float b = 0.5f * a - 0.5f;
    const float s = fminf(fmaxf(a * (float)i + b, 0.0f), (float)(src_len - 1u));
    const float x0 = floorf(s);
    const float frac = s - x0;
    x0s[i] = (int)x0;
    float w[6] = {hq_lanczos3(frac + 2.0f), hq_lanczos3(frac + 1.0f), hq_lanczos3(frac), hq_lanczos3(frac - 1.0f), hq_lanczos3(frac - 2.0f), hq_lanczos3(frac - 3.0f)};
    const float sum = w[0] + w[1] + w[2] + w[3] + w[4] + w[5];
    const float inv = __fdiv_rn(1.0f, sum);
#pragma unroll
    for (int t = 0; t < 6; ++t) wtab[i * 6u + t] = w[t] * inv;
}

// H pass: (sw, sh) -> (dw, sh);  V pass: (dw, sh) -> (dw, dh).  cuda/resize.rs:331-402
__global__ void __launch_bounds__(256) resize_lanczos_h_kernel(const float* __restrict__ src, float* __restrict__ inter, const int* __restrict__ x0s,
                                                               const float* __restrict__ wtab, uint32_t sw, uint32_t sh, uint32_t dw) {
    const uint32_t x = blockIdx.x * 32u + threadIdx.x, y = blockIdx.y * 8u + threadIdx.y;
    if (x >= dw || y >= sh) return;
    const float* row = src + ((size_t)blockIdx.z * sh + y) * sw * 3u;
    const int x0 = __ldg(x0s + x);
    const float* w = wtab + (size_t)x * 6u;
    float a0 = 0.0f, a1 = 0.0f, a2 = 0.0f;
#pragma unroll
    for (int t = 0; t < 6; ++t) {
        const float* p = row + (uint32_t)max(0, min(x0 + t - 2, (int)sw - 1)) * 3u;
        const float wt = __ldg(w + t);
        a0 = fmaf(wt, __ldg(p), a0); a1 = fmaf(wt, __ldg(p + 1), a1); a2 = fmaf(wt, __ldg(p + 2), a2);
    }
    float* o = inter + (((size_t)blockIdx.z * sh + y) * dw + x) * 3u;
    o[0] = a0; o[1] = a1; o[2] = a2;
}

__global__ void __launch_bounds__(256) resize_lanczos_v_kernel(const float* __restrict__ inter, float* __restrict__ dst, const int* __restrict__ y0s,
                                                               const float* __restrict__ wtab, uint32_t sh, uint32_t dw, uint32_t dh) {
    const uint32_t x = blockIdx.x * 32u + threadIdx.x, y = blockIdx.y * 8u + threadIdx.y;
    if (x >= dw || y >= dh) return;
    const float* img = inter + (size_t)blockIdx.z * sh * dw * 3u + (size_t)x * 3u;
    const int y0 = __ldg(y0s + y);
    const float* w = wtab + (size_t)y * 6u;
    float a0 = 0.0f, a1 = 0.0f, a2 = 0.0f;
#pragma unroll
    for (int t = 0; t < 6; ++t) {
        const float* p = img + (size_t)max(0, min(y0 + t - 2, (int)sh - 1)) * dw * 3u;
        const float wt = __ldg(w + t);
        a0 = fmaf(wt, __ldg(p), a0); a1 = fmaf(wt, __ldg(p + 1), a1); a2 = fmaf(wt, __ldg(p + 2), a2);
    }
    float* o = dst + (((size_t)blockIdx.z * dh + y) * dw + x) * 3u;
    o[0] = a0; o[1] = a1; o[2] = a2;
}

// ── warps ────────────────────────────────────────────────────────────────────────────────────
// Coordinates / validity exactly as the bilinear kernels (warp_common.cuh documents the rules); the samplers take the
// UNCLAMPED valid coordinate (cuda/warp_affine.rs:260-268, cuda/warp_perspective.rs:195-210).
template <bool PERSPECTIVE, bool LANCZOS>
__global__ void __launch_bounds__(256) warp_hq_kernel(const float* __restrict__ src, float* __restrict__ dst, uint32_t sw, uint32_t sh, uint32_t dw,
                                                      uint32_t dh, const __grid_constant__ HqMat M) {
    const uint32_t gx = blockIdx.x * 32u + threadIdx.x, gy = blockIdx.y * 8u + threadIdx.y;
    if (gx >= dw || gy >= dh) return;
    const float* s = src + (size_t)blockIdx.z * sw * sh * 3u;
    float* d = dst + ((size_t)blockIdx.z * dw * dh + (size_t)gy * dw + gx) * 3u;
    const float* m = M.m;
    float sx, sy;
    bool ok;
    if (PERSPECTIVE) {
        const float x = (float)gx, y = (float)gy;
        const float w = m[6] * x + m[7] * y + m[8];
        ok = !(fabsf(w) < 1e-10f);
        sx = __fdiv_rn(m[0] * x + m[1] * y + m[2], w);
        sy = __fdiv_rn(m[3] * x + m[4] * y + m[5], w);
        ok = ok && !(sx < 0.0f || sx >= (float)sw || sy < 0.0f || sy >= (float)sh);
    } else {
        const float sx0 = m[1] * (float)gy + m[2], sy0 = m[4] * (float)gy + m[5];
        sx = m[0] * (float)gx + sx0;
        sy = m[3] * (float)gx + sy0;
        const bool x_ok = (fabsf(m[0]) < 1e-6f) ? (sx0 >= 0.0f && sx0 < (float)sw) : (sx >= 0.0f && sx < (float)sw);
        const bool y_ok = (fabsf(m[3]) < 1e-6f) ? (sy0 >= 0.0f && sy0 < (float)sh) : (sy >= 0.0f && sy < (float)sh);
        ok = x_ok && y_ok;
    }
    float v[3] = {0.0f, 0.0f, 0.0f};
    if (ok) {
        if (LANCZOS) sample_lanczos_c3(s, sw, sh, sx, sy, v);
        else sample_bicubic_c3(s, sw, sh, sx, sy, v);
    }
    d[0] = v[0]; d[1] = v[1]; d[2] = v[2];
}

static inline void hq_coeffs(uint32_t src_len, uint32_t dst_len, float* a, float* b) {  // PixelMapping::HalfPixel
    *a = (float)src_len / (float)dst_len;
    *b = 0.5f * *a - 0.5f;
}

int launch_resize_bicubic_c3(cudaStream_t s, const float* src, float* dst, uint32_t sw, uint32_t sh, uint32_t dw, uint32_t dh, uint32_t batch) {
    float ax, bx, ay, by;
    hq_coeffs(sw, dw, &ax, &bx);
    hq_coeffs(sh, dh, &ay, &by);
    dim3 block(32, 8), grid(div_up(dw, 32), div_up(dh, 8), batch);
    resize_bicubic_c3_kernel<<<grid, block, 0, s>>>(src, dst, sw, sh, dw, dh, ax, bx, ay, by);
    return check_launch("resize_bicubic_c3_kernel");
}

template <bool PERSPECTIVE>
int launch_warp_hq(cudaStream_t s, const float* src, float* dst, uint32_t sw, uint32_t sh, uint32_t dw, uint32_t dh, uint32_t batch,
                   const float* minv, bool lanczos) {
    HqMat M;
    for (int i = 0; i < 9; ++i) M.m[i] = (PERSPECTIVE || i < 6) ? minv[i] : 0.0f;
    dim3 block(32, 8), grid(div_up(dw, 32), div_up(dh, 8), batch);
    if (lanczos) warp_hq_kernel<PERSPECTIVE, true><<<grid, block, 0, s>>>(src, dst, sw, sh, dw, dh, M);
    else warp_hq_kernel<PERSPECTIVE, false><<<grid, block, 0, s>>>(src, dst, sw, sh, dw, dh, M);
    return check_launch(lanczos ? "warp_lanczos_kernel" : "warp_bicubic_kernel");
}
template int launch_warp_hq<false>(cudaStream_t, const float*, float*, uint32_t, uint32_t, uint32_t, uint32_t, uint32_t, const float*, bool);
template int launch_warp_hq<true>(cudaStream_t, const float*, float*, uint32_t, uint32_t, uint32_t, uint32_t, uint32_t, const float*, bool);

}  // namespace kb200

using namespace kb200;

extern "C" {

KB200_API int kb200_resize_bicubic_f32_c3(kb200_stream_t stream, const float* src, size_t src_len, float* dst, size_t dst_len, uint32_t sw,
                                          uint32_t sh, uint32_t dw, uint32_t dh, uint32_t batch) {
    KB200_TRY(check_ptr("src", src)); KB200_TRY(check_ptr("dst", dst));
    KB200_TRY(check_geometry(sw, sh, dw, dh, batch));
    if (batch > 65535u) return fail(KB200_ERR_INVALID_ARGUMENT, "batch %u exceeds 65535 per call", batch);
    KB200_TRY(check_slice("dst", dst_len, (size_t)dw * dh * 3 * batch));
    KB200_TRY(check_slice("src", src_len, (size_t)sw * sh * 3 * batch));
    return launch_resize_bicubic_c3(as_stream(stream), src, dst, sw, sh, dw, dh, batch);
}

KB200_API size_t kb200_resize_lanczos_scratch_len(uint32_t sh, uint32_t dw, uint32_t dh, uint32_t batch) {
    // intermediate (dst_w x src_h x 3 per image) + the two axis tables (tap base + six weights per destination index)
    return (size_t)dw * sh * 3 * batch + 7 * ((size_t)dw + dh);
}

KB200_API int kb200_resize_lanczos_f32_c3(kb200_stream_t stream, const float* src, size_t src_len, float* dst, size_t dst_len, float* scratch,
                                          size_t scratch_len, uint32_t sw, uint32_t sh, uint32_t dw, uint32_t dh, uint32_t batch) {
    KB200_TRY(check_ptr("src", src)); KB200_TRY(check_ptr("dst", dst)); KB200_TRY(check_ptr("scratch", scratch));
    KB200_TRY(check_geometry(sw, sh, dw, dh, batch));
    if (batch > 65535u) return fail(KB200_ERR_INVALID_ARGUMENT, "batch %u exceeds 65535 per call", batch);
    KB200_TRY(check_slice("dst", dst_len, (size_t)dw * dh * 3 * batch));
    KB200_TRY(check_slice("src", src_len, (size_t)sw * sh * 3 * batch));
    KB200_TRY(check_slice("scratch", scratch_len, kb200_resize_lanczos_scratch_len(sh, dw, dh, batch)));
    cudaStream_t s = as_stream(stream);
    float* inter = scratch;
    float* wx = inter + (size_t)dw * sh * 3 * batch;
    float* wy = wx + (size_t)dw * 6;
    int* x0s = reinterpret_cast<int*>(wy + (size_t)dh * 6);
    int* y0s = x0s + dw;
    lanczos_axis_kernel<<<div_up(dw, 128), 128, 0, s>>>(sw, dw, x0s, wx);
    lanczos_axis_kernel<<<div_up(dh, 128), 128, 0, s>>>(sh, dh, y0s, wy);
    dim3 block(32, 8);
    resize_lanczos_h_kernel<<<dim3(div_up(dw, 32), div_up(sh, 8), batch), block, 0, s>>>(src, inter, x0s, wx, sw, sh, dw);
    resize_lanczos_v_kernel<<<dim3(div_up(dw, 32), div_up(dh, 8), batch), block, 0, s>>>(inter, dst, y0s, wy, sh, dw, dh);
    return check_launch("resize_lanczos_kernels");
}

}  // extern "C"
