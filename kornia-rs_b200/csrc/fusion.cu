// fusion.cu — the reference's fusion-engine stage vocabulary as PRE-INSTANTIATED pipelines (SURVEY §8(f) #3).
//
// Reference: cuda/fusion.rs — an NVRTC code generator that composes per-op snippets (source -> maps -> sink) into one
// kernel with register value flow and all parameters in a `__grid_constant__` blob.  Its stage library on this path:
//   ReadU8RgbBilinear (:520-585)  u8 HWC source sampled at the half-pixel coordinate `a*d + b` (max 0), weights first
//   Normalize (:592-620)          v * scale[c] + bias[c]
//   RgbToGray (:624-642)          0.299 x + 0.587 y + 0.114 z, replicated to the three lanes
//   WriteChwF32 / WriteC1F32 (:645-690)  three planes / the .x lane
// There is no runtime compiler in this library (everything is AOT sm_90a code), so the composable shapes are compiled
// ahead of time as template instantiations of one kernel: map chains {}, {N}, {G}, {N,G}, {G,N} x sinks {CHW, C1} — every
// chain the vocabulary can express without repeating a stage.  Same contract as the engine: f32 register flow between
// stages (NOT bit-equal to running the ops through u8 buffers, fusion.rs:21-27), parameters in the constant bank, batch
// as grid.z with per-image outputs at z * out_elems (FKL "DivergentBatch", :269-283) — here over one strided source
// buffer.  Arithmetic = the generated kernel's (unfused under -fmad=false), bit-exact with the engine's output.
#include "kb200_common.cuh"

namespace kb200 {

struct FusionArgs {
    uint32_t sw, sh, dw, dh;
    float ax, bx, ay, by;
    float scale[3], bias[3];
};

enum { FUS_NONE = 0, FUS_NORM = 1, FUS_GRAY = 2, FUS_NORM_GRAY = 3, FUS_GRAY_NORM = 4 };

template <int MAPS, int SINK>
__global__ void __launch_bounds__(256) fused_pipeline_kernel(const uint8_t* __restrict__ src, float* __restrict__ dst, const __grid_constant__ FusionArgs P) {
    const uint32_t x = blockIdx.x * 32u + threadIdx.x, y = blockIdx.y * 8u + threadIdx.y;
    if (x >= P.dw || y >= P.dh) return;
    const uint8_t* s = src + (size_t)blockIdx.z * P.sw * P.sh * 3u;
    const size_t plane = (size_t)P.dw * P.dh;
    float* d = dst + (size_t)blockIdx.z * plane * (SINK == 0 ? 3u : 1u);
    // stage 0: ReadU8RgbBilinear
    const float sxf = fmaxf(P.ax * (float)x + P.bx, 0.0f), syf = fmaxf(P.ay * (float)y + P.by, 0.0f);
    const uint32_t sx0 = min((uint32_t)sxf, P.sw - 1u), sy0 = min((uint32_t)syf, P.sh - 1u);
    const uint32_t sx1 = min(sx0 + 1u, P.sw - 1u), sy1 = min(sy0 + 1u, P.sh - 1u);
    const float wx = sxf - (float)sx0, wy = syf - (float)sy0;
    const uint8_t* r0 = s + (size_t)sy0 * P.sw * 3u;
    const uint8_t* r1 = s + (size_t)sy1 * P.sw * 3u;
    const float w00 = (1.0f - wy) * (1.0f - wx), w01 = (1.0f - wy) * wx, w10 = wy * (1.0f - wx), w11 = wy * wx;
    float v[3];
#pragma unroll
    for (int c = 0; c < 3; ++c)
        v[c] = w00 * (float)r0[sx0 * 3u + c] + w01 * (float)r0[sx1 * 3u + c] + w10 * (float)r1[sx0 * 3u + c] + w11 * (float)r1[sx1 * 3u + c];
    auto norm = [&]() {
#pragma unroll
        for (int c = 0; c < 3; ++c) v[c] = v[c] * P.scale[c] + P.bias[c];
    };
    auto gray = [&]() { const float g = 0.299f * v[0] + 0.587f * v[1] + 0.114f * v[2]; v[0] = g; v[1] = g; v[2] = g; };
    if (MAPS == FUS_NORM) norm();
    else if (MAPS == FUS_GRAY) gray();
    else if (MAPS == FUS_NORM_GRAY) { norm(); gray(); }
    else if (MAPS == FUS_GRAY_NORM) { gray(); norm(); }
    const size_t di = (size_t)y * P.dw + x;
    if (SINK == 0) { d[di] = v[0]; d[di + plane] = v[1]; d[di + 2u * plane] = v[2]; }
    else d[di] = v[0];
}

template <int MAPS>
static void fusion_launch(int sink, dim3 grid, cudaStream_t s, const uint8_t* src, float* dst, const FusionArgs& P) {
    if (sink == 0) fused_pipeline_kernel<MAPS, 0><<<grid, dim3(32, 8), 0, s>>>(src, dst, P);
    else fused_pipeline_kernel<MAPS, 1><<<grid, dim3(32, 8), 0, s>>>(src, dst, P);
}

}  // namespace kb200

using namespace kb200;

extern "C" {

KB200_API int kb200_fused_pipeline_u8_f32(kb200_stream_t stream, const uint8_t* src, size_t src_len, float* dst, size_t dst_len, uint32_t sw,
                                          uint32_t sh, uint32_t dw, uint32_t dh, uint32_t batch, int maps, const float scale[3],
                                          const float bias[3], int sink) {
    KB200_TRY(check_ptr("src", src)); KB200_TRY(check_ptr("dst", dst));
    KB200_TRY(check_geometry(sw, sh, dw, dh, batch));
    if (batch > 65535u) return fail(KB200_ERR_INVALID_ARGUMENT, "batch %u exceeds 65535 per call", batch);
    if (maps < FUS_NONE || maps > FUS_GRAY_NORM)
        return fail(KB200_ERR_UNSUPPORTED, "invalid pipeline: map chain %d is not one of the pre-instantiated shapes", maps);   // FusionError::Pipeline
    if (sink != 0 && sink != 1) return fail(KB200_ERR_UNSUPPORTED, "invalid pipeline: unknown sink %d", sink);
    const bool has_norm = maps == FUS_NORM || maps == FUS_NORM_GRAY || maps == FUS_GRAY_NORM;
    if (has_norm) { KB200_TRY(check_ptr("scale", scale)); KB200_TRY(check_ptr("bias", bias)); }
    KB200_TRY(check_slice("src", src_len, (size_t)sw * sh * 3 * batch));                       // src_bytes_required
    KB200_TRY(check_slice("dst", dst_len, (size_t)dw * dh * (sink == 0 ? 3 : 1) * batch));     // out_elems
    FusionArgs P;
    P.sw = sw; P.sh = sh; P.dw = dw; P.dh = dh;
    P.ax = (float)sw / (float)dw; P.ay = (float)sh / (float)dh;      // fusion.rs:541-546
    P.bx = 0.5f * P.ax - 0.5f; P.by = 0.5f * P.ay - 0.5f;
    for (int c = 0; c < 3; ++c) { P.scale[c] = has_norm ? scale[c] : 1.0f; P.bias[c] = has_norm ? bias[c] : 0.0f; }
    dim3 grid(div_up(dw, 32), div_up(dh, 8), batch);
    cudaStream_t s = as_stream(stream);
    switch (maps) {
        case FUS_NONE: fusion_launch<FUS_NONE>(sink, grid, s, src, dst, P); break;
        case FUS_NORM: fusion_launch<FUS_NORM>(sink, grid, s, src, dst, P); break;
        case FUS_GRAY: fusion_launch<FUS_GRAY>(sink, grid, s, src, dst, P); break;
        case FUS_NORM_GRAY: fusion_launch<FUS_NORM_GRAY>(sink, grid, s, src, dst, P); break;
        default: fusion_launch<FUS_GRAY_NORM>(sink, grid, s, src, dst, P); break;
    }
    return check_launch("fused_pipeline_kernel");
}

}  // extern "C"
