// point_ceiling.cu — bandwidth probes for the fused resize headline's own traffic (tools/point_ceiling.py builds this
// with nvcc into a temporary directory; it is not part of the library).
//
// The headline reads 1 of every `period` source rows (row period*d + first) and writes three f32 planes of dw x dh.
// Every probe walks one (image, destination row) per CTA of 256 threads with 16-byte accesses:
//   probe_read   reads the tapped rows only (LDG.128), folds them into one word that is stored only if it hits a
//                value the data cannot produce, so the loads stay live and nothing is written
//   probe_write  writes every destination value (STG.128), reads nothing
//   probe_twin   reads the tapped row into shared memory (LDG.128), writes (float)byte of the point taps, lane-contiguous
//                STG.128 per plane: the headline's traffic with no arithmetic
//   probe_memcpy cudaMemcpyAsync device to device
#include <cuda_runtime.h>
#include <stdint.h>

namespace {

constexpr int kThreads = 256;

__device__ __forceinline__ uint4 ldg_nc(const uint4* p) {
    uint4 v;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
    return v;
}

struct Geo {
    uint32_t sh, row_bytes, dw, dh, period, first;
};

__global__ void __launch_bounds__(kThreads) read_kernel(const uint8_t* __restrict__ src, uint32_t* __restrict__ sink, Geo g) {
    const uint32_t dy = blockIdx.x, img = blockIdx.y;
    const uint4* row = reinterpret_cast<const uint4*>(src + ((size_t)img * g.sh + (size_t)dy * g.period + g.first) * g.row_bytes);
    uint32_t acc = 0;
    for (uint32_t i = threadIdx.x; i < g.row_bytes / 16u; i += kThreads) {
        const uint4 v = ldg_nc(row + i);
        acc ^= v.x ^ (v.y * 3u) ^ (v.z * 5u) ^ (v.w * 7u);
    }
    if (acc == 0x9E3779B9u && threadIdx.x == 1000u) *sink = acc;   // threadIdx.x < 256: never stores
}

__global__ void __launch_bounds__(kThreads) write_kernel(float* __restrict__ dst, Geo g) {
    const uint32_t dy = blockIdx.x, img = blockIdx.y;
    const size_t plane = (size_t)g.dw * g.dh;
    const float v = (float)dy;
    for (uint32_t c = 0; c < 3; ++c) {
        float4* out = reinterpret_cast<float4*>(dst + ((size_t)img * 3 + c) * plane + (size_t)dy * g.dw);
        for (uint32_t i = threadIdx.x; i < g.dw / 4u; i += kThreads) out[i] = make_float4(v, v, v, v);
    }
}

__global__ void __launch_bounds__(kThreads) twin_kernel(const uint8_t* __restrict__ src, float* __restrict__ dst, Geo g) {
    extern __shared__ __align__(16) uint8_t row_s[];
    const uint32_t dy = blockIdx.x, img = blockIdx.y;
    const uint4* row = reinterpret_cast<const uint4*>(src + ((size_t)img * g.sh + (size_t)dy * g.period + g.first) * g.row_bytes);
    for (uint32_t i = threadIdx.x; i < g.row_bytes / 16u; i += kThreads) reinterpret_cast<uint4*>(row_s)[i] = ldg_nc(row + i);
    __syncthreads();
    const size_t plane = (size_t)g.dw * g.dh;
    // destination column x taps source column period*x + first (the 3:1 point sampler: (x+0.5)*3-0.5 = 3x+1)
    for (uint32_t c = 0; c < 3; ++c) {
        float4* out = reinterpret_cast<float4*>(dst + ((size_t)img * 3 + c) * plane + (size_t)dy * g.dw);
        for (uint32_t i = threadIdx.x; i < g.dw / 4u; i += kThreads) {
            const uint8_t* t = row_s + (size_t)(4u * i * g.period + g.first) * 3u + c;
            const uint32_t s = g.period * 3u;
            out[i] = make_float4((float)t[0], (float)t[s], (float)t[2u * s], (float)t[3u * s]);
        }
    }
}

}  // namespace

extern "C" {

int probe_read(const uint8_t* src, uint32_t* sink, uint32_t batch, uint32_t sh, uint32_t row_bytes, uint32_t dh, uint32_t period,
               uint32_t first, cudaStream_t s) {
    read_kernel<<<dim3(dh, batch), kThreads, 0, s>>>(src, sink, Geo{sh, row_bytes, 0, dh, period, first});
    return (int)cudaGetLastError();
}

int probe_write(float* dst, uint32_t batch, uint32_t dw, uint32_t dh, cudaStream_t s) {
    write_kernel<<<dim3(dh, batch), kThreads, 0, s>>>(dst, Geo{0, 0, dw, dh, 1, 0});
    return (int)cudaGetLastError();
}

int probe_twin(const uint8_t* src, float* dst, uint32_t batch, uint32_t sh, uint32_t row_bytes, uint32_t dw, uint32_t dh, uint32_t period,
               uint32_t first, cudaStream_t s) {
    twin_kernel<<<dim3(dh, batch), kThreads, row_bytes, s>>>(src, dst, Geo{sh, row_bytes, dw, dh, period, first});
    return (int)cudaGetLastError();
}

int probe_memcpy(void* dst, const void* src, size_t bytes, cudaStream_t s) {
    return (int)cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, s);
}

}  // extern "C"
