// host_pipeline.cu — the HOST-buffer form of the hot path.
//
// The reference's fused resize (`resize_normalize_to_tensor_u8_to_f32_bilinear`, resize/fused.rs:147) takes host
// images and writes a host tensor.  A drop-in for that call therefore has to move the frames over PCIe, and at 4K the
// link — not the kernel — sets the rate (a 64-frame 4K batch is 1.59 GB in, 0.71 GB out; the kernel needs < 1 ms).
// Two things keep the link busy and lightly loaded:
//
//   * a ring of `depth` streams, each owning a device source and destination staging buffer: chunk i's upload, kernel
//     and download run on stream i mod depth, so uploads (H2D engine), kernels and downloads (D2H engine) of
//     neighbouring chunks overlap.  Nothing is allocated or synchronised per call; the call only ENQUEUES, fenced
//     against the caller's stream with events (same contract as every device-buffer entry point).
//   * rows no destination row taps are never uploaded.  For an integer downscale the tapped rows are periodic
//     (resize_row_plan); one strided 2-D copy per chunk (cudaMemcpy2DAsync: pitch = period rows, width = keep rows)
//     lands them compacted, and the kernel reads them through the row map (FusedParams::row_p/f/k).  At 2160 -> 720
//     the vertical weight is exactly 0, one source row in three is needed, and the upload shrinks 3x.
#include <vector>

#include "kb200_common.cuh"
#include "resize_fused.cuh"

struct kb200_host_pipeline {
    int device = 0;
    int depth = 0;
    size_t src_bytes = 0, dst_bytes = 0;  // per staging buffer
    std::vector<cudaStream_t> streams;
    std::vector<uint8_t*> src;
    std::vector<uint8_t*> dst;
    std::vector<cudaEvent_t> done;
    cudaEvent_t start = nullptr;
    uint64_t h2d_bytes = 0, d2h_bytes = 0;  // of the last call
};

using namespace kb200;

namespace kb200 {   // preprocess.cu
int preprocess_validate(const kb200_preprocess_desc* desc);
size_t preprocess_frame_bytes(const kb200_preprocess_desc& d);
int preprocess_launch_strided(cudaStream_t s, const kb200_preprocess_desc& d, const uint8_t* base, size_t stride, uint32_t batch, void* dst, int out);
}

namespace {

int cuda_fail(const char* what, cudaError_t e) { return fail(KB200_ERR_CUDA, "%s failed: %s", what, cudaGetErrorString(e)); }

#define KB200_CUDA(call)                                   \
    do {                                                   \
        cudaError_t e__ = (call);                          \
        if (e__ != cudaSuccess) return cuda_fail(#call, e__); \
    } while (0)

void destroy(kb200_host_pipeline* p) {
    if (!p) return;
    int prev = -1;
    cudaGetDevice(&prev);
    cudaSetDevice(p->device);
    for (auto s : p->streams) if (s) { cudaStreamSynchronize(s); cudaStreamDestroy(s); }
    for (auto b : p->src) if (b) cudaFree(b);
    for (auto b : p->dst) if (b) cudaFree(b);
    for (auto e : p->done) if (e) cudaEventDestroy(e);
    if (p->start) cudaEventDestroy(p->start);
    if (prev >= 0) cudaSetDevice(prev);
    delete p;
}

}  // namespace

extern "C" {

KB200_API int kb200_host_pipeline_create(int device, size_t src_chunk_bytes, size_t dst_chunk_bytes, int depth,
                                         kb200_host_pipeline** out) {
    KB200_TRY(check_ptr("out", out));
    *out = nullptr;
    if (depth < 1 || depth > 8) return fail(KB200_ERR_INVALID_ARGUMENT, "pipeline depth %d outside 1..8", depth);
    if (src_chunk_bytes == 0 || dst_chunk_bytes == 0) return fail(KB200_ERR_INVALID_ARGUMENT, "staging sizes must be non-zero");
    KB200_CUDA(cudaSetDevice(device));
    kb200_host_pipeline* p = new kb200_host_pipeline();
    p->device = device; p->depth = depth;
    p->src_bytes = (src_chunk_bytes + 255) & ~(size_t)255;
    p->dst_bytes = (dst_chunk_bytes + 255) & ~(size_t)255;
    p->streams.assign(depth, nullptr); p->src.assign(depth, nullptr); p->dst.assign(depth, nullptr); p->done.assign(depth, nullptr);
    cudaError_t e = cudaEventCreateWithFlags(&p->start, cudaEventDisableTiming);
    for (int i = 0; i < depth && e == cudaSuccess; ++i) {
        e = cudaStreamCreateWithFlags(&p->streams[i], cudaStreamNonBlocking);
        if (e == cudaSuccess) e = cudaMalloc(&p->src[i], p->src_bytes);
        if (e == cudaSuccess) e = cudaMalloc(&p->dst[i], p->dst_bytes);
        if (e == cudaSuccess) e = cudaEventCreateWithFlags(&p->done[i], cudaEventDisableTiming);
    }
    if (e != cudaSuccess) { destroy(p); return cuda_fail("kb200_host_pipeline_create", e); }
    *out = p;
    return KB200_OK;
}

KB200_API void kb200_host_pipeline_destroy(kb200_host_pipeline* p) { destroy(p); }

KB200_API int kb200_host_pipeline_last_transfer(const kb200_host_pipeline* p, uint64_t* h2d_bytes, uint64_t* d2h_bytes) {
    KB200_TRY(check_ptr("pipeline", p));
    if (h2d_bytes) *h2d_bytes = p->h2d_bytes;
    if (d2h_bytes) *d2h_bytes = p->d2h_bytes;
    return KB200_OK;
}

KB200_API int kb200_host_register(void* ptr, size_t bytes) {
    KB200_TRY(check_ptr("ptr", ptr));
    KB200_CUDA(cudaHostRegister(ptr, bytes, cudaHostRegisterDefault));
    return KB200_OK;
}

KB200_API int kb200_host_unregister(void* ptr) {
    KB200_TRY(check_ptr("ptr", ptr));
    KB200_CUDA(cudaHostUnregister(ptr));
    return KB200_OK;
}

KB200_API int kb200_resize_normalize_chw_u8_host(kb200_host_pipeline* pipe, kb200_stream_t stream, const uint8_t* host_src,
                                                 size_t src_len, void* host_dst, size_t dst_len, uint32_t sw, uint32_t sh,
                                                 uint32_t dw, uint32_t dh, uint32_t batch, const float scale[3],
                                                 const float bias[3], int leaf, int out_format) {
    KB200_TRY(check_ptr("pipeline", pipe));
    KB200_TRY(check_ptr("src", host_src)); KB200_TRY(check_ptr("dst", host_dst));
    KB200_TRY(check_ptr("scale", scale)); KB200_TRY(check_ptr("bias", bias));
    if (leaf < 0 || leaf > 2) return fail(KB200_ERR_INVALID_ARGUMENT, "unknown cpu leaf %d", leaf);
    if (out_format != KB200_OUT_F32 && out_format != KB200_OUT_F16 && out_format != KB200_OUT_BF16)
        return fail(KB200_ERR_INVALID_ARGUMENT, "unknown output format %d", out_format);
    if (batch == 0) return fail(KB200_ERR_INVALID_ARGUMENT, "batch must be non-zero");
    KB200_TRY(check_slice("src", src_len, (size_t)sw * sh * 3 * batch));
    KB200_TRY(check_slice("dst", dst_len, (size_t)dw * dh * 3 * batch));
    pipe->h2d_bytes = pipe->d2h_bytes = 0;
    if (dw == 0 || dh == 0 || sw == 0 || sh == 0) return KB200_OK;  // resize/fused.rs:184-186
    KB200_CUDA(cudaSetDevice(pipe->device));

    FusedParams p = make_fused_params(sw, sh, dw, dh, scale, bias, leaf);
    resize_row_plan(sh, dh, &p.row_p, &p.row_f, &p.row_k);
    p.src_rows = sh / p.row_p * p.row_k;
    const size_t row_bytes = (size_t)sw * 3;
    const size_t src_frame_dev = row_bytes * p.src_rows;          // compacted frame in the staging buffer
    const size_t src_frame_host = row_bytes * sh;
    const size_t dst_frame = (size_t)dw * dh * 3 * (out_format == KB200_OUT_F32 ? sizeof(float) : sizeof(uint16_t));
    const size_t per_chunk = std::min<size_t>(std::min(pipe->src_bytes / src_frame_dev, pipe->dst_bytes / dst_frame), 65535);
    if (per_chunk == 0)
        return fail(KB200_ERR_INVALID_ARGUMENT, "pipeline staging (%zu B src, %zu B dst) is smaller than one frame (%zu B, %zu B)",
                    pipe->src_bytes, pipe->dst_bytes, src_frame_dev, dst_frame);

    cudaStream_t user = as_stream(stream);
    KB200_CUDA(cudaEventRecord(pipe->start, user));
    for (int k = 0; k < pipe->depth; ++k) KB200_CUDA(cudaStreamWaitEvent(pipe->streams[k], pipe->start, 0));
    uint32_t f0 = 0;
    int used = 0;
    for (uint32_t ci = 0; f0 < batch; ++ci) {
        const int k = (int)(ci % (uint32_t)pipe->depth);
        used = std::max(used, k + 1);
        const uint32_t n = (uint32_t)std::min<size_t>(per_chunk, batch - f0);
        cudaStream_t s = pipe->streams[k];
        const uint8_t* hs = host_src + (size_t)f0 * src_frame_host;
        if (p.row_p == 1) {
            KB200_CUDA(cudaMemcpyAsync(pipe->src[k], hs, src_frame_host * n, cudaMemcpyHostToDevice, s));
        } else {
            // frames are contiguous on the host and sh % period == 0, so the whole chunk is ONE strided copy:
            // `n * sh / period` groups, each `keep` rows wide, `period` rows apart
            KB200_CUDA(cudaMemcpy2DAsync(pipe->src[k], row_bytes * p.row_k, hs + row_bytes * p.row_f, row_bytes * p.row_p,
                                         row_bytes * p.row_k, (size_t)n * (sh / p.row_p), cudaMemcpyHostToDevice, s));
        }
        if (out_format == KB200_OUT_F32) KB200_TRY(launch_fused_resize(s, pipe->src[k], reinterpret_cast<float*>(pipe->dst[k]), p, n));
        else if (out_format == KB200_OUT_F16) KB200_TRY(launch_fused_resize(s, pipe->src[k], reinterpret_cast<__half*>(pipe->dst[k]), p, n));
        else KB200_TRY(launch_fused_resize(s, pipe->src[k], reinterpret_cast<__nv_bfloat16*>(pipe->dst[k]), p, n));
        KB200_CUDA(cudaMemcpyAsync(static_cast<uint8_t*>(host_dst) + (size_t)f0 * dst_frame, pipe->dst[k], dst_frame * n,
                                   cudaMemcpyDeviceToHost, s));
        pipe->h2d_bytes += src_frame_dev * n;
        pipe->d2h_bytes += dst_frame * n;
        f0 += n;
    }
    for (int k = 0; k < used; ++k) {
        KB200_CUDA(cudaEventRecord(pipe->done[k], pipe->streams[k]));
        KB200_CUDA(cudaStreamWaitEvent(user, pipe->done[k], 0));
    }
    return KB200_OK;
}

KB200_API int kb200_resize_normalize_chw_u8_f32_host(kb200_host_pipeline* pipe, kb200_stream_t stream,
                                                     const uint8_t* host_src, size_t src_len, float* host_dst,
                                                     size_t dst_len, uint32_t sw, uint32_t sh, uint32_t dw, uint32_t dh,
                                                     uint32_t batch, const float scale[3], const float bias[3], int leaf) {
    return kb200_resize_normalize_chw_u8_host(pipe, stream, host_src, src_len, host_dst, dst_len, sw, sh, dw, dh, batch, scale, bias,
                                              leaf, KB200_OUT_F32);
}

// Host-buffer form of Preprocessor::run_raw_batch (preprocess.rs:1234; the reference's Python Preprocessor pins and
// uploads camera frames itself, kornia-py/src/cuda_ext/mod.rs:700-760): `batch` raw frames at host_base + i*frame_stride
// (page-locked memory for overlap) -> host tensor [batch,3,dst_h,dst_w] of `out_format` (f32, binary16 or bfloat16).  Chunks
// of frames ride the same stream ring as the fused resize: upload -> fused preprocess kernel (one launch per chunk) -> download.
KB200_API int kb200_preprocess_host_format(kb200_host_pipeline* pipe, kb200_stream_t stream, const kb200_preprocess_desc* desc,
                                           const uint8_t* host_base, size_t base_len, size_t frame_stride, uint32_t batch,
                                           void* host_dst, size_t dst_len, int out_format) {
    KB200_TRY(check_ptr("pipeline", pipe));
    KB200_TRY(preprocess_validate(desc));
    KB200_TRY(check_ptr("base", host_base)); KB200_TRY(check_ptr("dst", host_dst));
    if (out_format != KB200_OUT_F32 && out_format != KB200_OUT_F16 && out_format != KB200_OUT_BF16)
        return fail(KB200_ERR_INVALID_ARGUMENT, "unknown output format %d", out_format);
    if (batch == 0) return fail(KB200_ERR_INVALID_ARGUMENT, "batch must be non-zero");
    const size_t need = preprocess_frame_bytes(*desc);
    if (frame_stride < need && batch > 1) return fail(KB200_ERR_INVALID_SOURCE, "frame stride %zu smaller than a frame (%zu bytes)", frame_stride, need);
    if (base_len < (size_t)(batch - 1) * frame_stride + need)
        return fail(KB200_ERR_INVALID_SOURCE, "invalid raw source at %dx%d (got %zu bytes, need %zu)", desc->src_w, desc->src_h, base_len,
                    (size_t)(batch - 1) * frame_stride + need);
    const size_t dst_frame_elems = (size_t)3 * desc->dst_w * desc->dst_h;
    KB200_TRY(check_slice("dst", dst_len, dst_frame_elems * batch));
    pipe->h2d_bytes = pipe->d2h_bytes = 0;
    KB200_CUDA(cudaSetDevice(pipe->device));
    const size_t elem = out_format == KB200_OUT_F32 ? sizeof(float) : sizeof(uint16_t);
    const size_t dst_frame = dst_frame_elems * elem;
    const size_t dev_stride = (need + 15) & ~(size_t)15;      // staged frames 16-byte aligned (the NV12 fast paths want aligned bases)
    const size_t per_chunk = std::min<size_t>(std::min(pipe->src_bytes / dev_stride, pipe->dst_bytes / dst_frame), 256);
    if (per_chunk == 0)
        return fail(KB200_ERR_INVALID_ARGUMENT, "pipeline staging (%zu B src, %zu B dst) is smaller than one frame (%zu B, %zu B)", pipe->src_bytes,
                    pipe->dst_bytes, dev_stride, dst_frame);
    cudaStream_t user = as_stream(stream);
    KB200_CUDA(cudaEventRecord(pipe->start, user));
    for (int k = 0; k < pipe->depth; ++k) KB200_CUDA(cudaStreamWaitEvent(pipe->streams[k], pipe->start, 0));
    uint32_t f0 = 0;
    int used = 0;
    for (uint32_t ci = 0; f0 < batch; ++ci) {
        const int k = (int)(ci % (uint32_t)pipe->depth);
        used = std::max(used, k + 1);
        const uint32_t n = (uint32_t)std::min<size_t>(per_chunk, batch - f0);
        cudaStream_t s = pipe->streams[k];
        const uint8_t* hs = host_base + (size_t)f0 * frame_stride;
        if (frame_stride == need && dev_stride == need) KB200_CUDA(cudaMemcpyAsync(pipe->src[k], hs, need * n, cudaMemcpyHostToDevice, s));
        else KB200_CUDA(cudaMemcpy2DAsync(pipe->src[k], dev_stride, hs, frame_stride, need, n, cudaMemcpyHostToDevice, s));
        KB200_TRY(preprocess_launch_strided(s, *desc, pipe->src[k], dev_stride, n, pipe->dst[k], out_format));
        KB200_CUDA(cudaMemcpyAsync(static_cast<uint8_t*>(host_dst) + (size_t)f0 * dst_frame, pipe->dst[k], dst_frame * n, cudaMemcpyDeviceToHost, s));
        pipe->h2d_bytes += need * n;
        pipe->d2h_bytes += dst_frame * n;
        f0 += n;
    }
    for (int k = 0; k < used; ++k) {
        KB200_CUDA(cudaEventRecord(pipe->done[k], pipe->streams[k]));
        KB200_CUDA(cudaStreamWaitEvent(user, pipe->done[k], 0));
    }
    return KB200_OK;
}

KB200_API int kb200_preprocess_host(kb200_host_pipeline* pipe, kb200_stream_t stream, const kb200_preprocess_desc* desc,
                                    const uint8_t* host_base, size_t base_len, size_t frame_stride, uint32_t batch, void* host_dst,
                                    size_t dst_len, int out_f16) {
    return kb200_preprocess_host_format(pipe, stream, desc, host_base, base_len, frame_stride, batch, host_dst, dst_len,
                                        out_f16 ? KB200_OUT_F16 : KB200_OUT_F32);
}

}  // extern "C"
