// resize_fused.cuh — parameter block and launcher of the fused u8 HWC -> f32 / f16 / bf16 CHW resize+normalize, shared
// between the device-buffer entry points (resize_fused.cu) and the host-buffer pipeline (host_pipeline.cu).
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "kb200_common.cuh"

namespace kb200 {

struct FusedParams {
    uint32_t sw, sh, dw, dh;
    float scale_x, scale_y;
    float scale[3], bias[3];
    uint32_t fma_bulk;
    // Row map of the source buffer.  Dense (1, 0, 1): row y of an image is row y of the buffer.  Compacted
    // (period P, first F, keep K): the buffer holds only rows with F <= y mod P < F + K, in order — what a strided
    // host->device copy of an integer downscale uploads.  src_rows = rows per image in the buffer.
    uint32_t row_p, row_f, row_k, src_rows;
};

__host__ __device__ __forceinline__ uint32_t fused_row_slot(const FusedParams& p, uint32_t y) {
    return p.row_p == 1u ? y : (y / p.row_p) * p.row_k + (y % p.row_p - p.row_f);
}

FusedParams make_fused_params(uint32_t sw, uint32_t sh, uint32_t dw, uint32_t dh, const float scale[3], const float bias[3], int leaf);
void resize_row_plan(uint32_t sh, uint32_t dh, uint32_t* period, uint32_t* first, uint32_t* keep);
// T = float, __half or __nv_bfloat16 (instantiated in resize_fused.cu); a 16-bit T is RNE(the f32 result).
template <typename T>
int launch_fused_resize(cudaStream_t s, const uint8_t* src, T* dst, const FusedParams& p, uint32_t batch);

}  // namespace kb200
