// resize_rows.cu — f32 HWC C=3 bilinear resize (a1), row-streaming design.
//
// Reference: resize/mod.rs:114-207 (CPU `resize`), interpolation/bilinear.rs:16-66, GPU twin cuda/resize.rs:97-235.
// The reference's GPU kernel is one thread per destination pixel with 12 scalar `__ldg` taps at a 12-byte lane stride
// and three 4-byte stores per pixel.  Here nothing in the inner loop touches global memory with scalar accesses:
//
//   * work unit = (image, tile of TW = 128*NPX destination columns, chunk of destination rows); persistent CTAs walk
//     their units with carry arithmetic.
//   * per destination row the TWO source rows it taps (y0, y1) are copied — only the float span the column tile
//     touches, rounded out to 16 B — global -> shared by the TMA engine (`cp.async.bulk`, SASS UBLKCP) into a short
//     mbarrier ring filled by a producer lane; every source byte is fetched once per column tile, in whole lines.
//     Zero-weight taps ARE fetched (f32 sources may hold inf/NaN and 0*inf must stay NaN, unlike the u8 fused path).
//   * 4 consumer warps; a thread owns NPX lane-contiguous destination columns for the whole unit: the x-side of the
//     sampler (x0/x1 offsets inside the span, fx, 1-fx) lives in registers, the y-side (fy, 1-fy) is published once per
//     stage by the producer.  Taps are 12 `LDS.32` at an odd word stride (conflict-free at 3:1 and 1:1).
//   * results go to a double-buffered shared-memory row and leave as lane-contiguous `STG.128` (a warp writes 512
//     contiguous bytes per instruction) instead of 12-byte-strided scalar stores.
//
// Arithmetic is the reference's expression tree (weights first, four terms summed left to right, unfused: this file is
// compiled with -fmad=false) — bit-identical to resize_f32_c3_kernel, which stays as the fallback for geometries the
// staging cannot take (rows not 16-byte aligned, destination width not a multiple of 4, nearest).
#include <algorithm>
#include <cmath>

#include "kb200_common.cuh"
#include "tma_ring.cuh"

namespace kb200 {

static constexpr int RR_CT = 128;              // consumer threads
static constexpr int RR_THREADS = RR_CT + 32;  // + producer warp
static constexpr int RR_MAX_STAGES = 8;

struct ResizeRowsParams {
    uint32_t sw, sh, dw, dh;
    float ax, bx, ay, by;          // PixelMapping::coeffs (cuda/resize.rs:462-478)
    float mean[3], inv_std[3];     // MODE 2 only
    uint32_t tiles_x, chunks_y, rows_per_chunk, nunits;
    uint32_t slot_floats;          // floats reserved per staged source-row span (multiple of 32)
    uint32_t row_floats;           // sw * 3
    uint32_t stages;
    uint32_t dtx, dcy, dimg;       // CTA stride decomposed for the carry walk
};

// source coordinate of one axis — cuda/resize.rs:113-125: clamp(a*i + b, 0, len-1), trunc, +1 tap clamped
__device__ __forceinline__ void rr_axis(uint32_t i, float a, float b, uint32_t len, uint32_t* i0, uint32_t* i1, float* f) {
    const float s = fmaxf(fminf(a * (float)i + b, (float)(len - 1u)), 0.0f);
    const uint32_t k = (uint32_t)s;
    *i0 = k;
    *i1 = min(k + 1u, len - 1u);
    *f = s - (float)k;
}

struct RRWalk {
    uint32_t tx, cy, img;
    __device__ __forceinline__ void init(uint32_t u, const ResizeRowsParams& P) {
        const uint32_t per_img = P.tiles_x * P.chunks_y;
        img = u / per_img;
        const uint32_t t = u - img * per_img;
        cy = t / P.tiles_x;
        tx = t - cy * P.tiles_x;
    }
    __device__ __forceinline__ void advance(const ResizeRowsParams& P) {
        tx += P.dtx; cy += P.dcy; img += P.dimg;
        if (tx >= P.tiles_x) { tx -= P.tiles_x; ++cy; }
        if (cy >= P.chunks_y) { cy -= P.chunks_y; ++img; }
        if (cy >= P.chunks_y) { cy -= P.chunks_y; ++img; }
    }
};

// span of source floats a column tile taps: [b0, b1), 4-float aligned (row_floats % 4 == 0)
__device__ __forceinline__ void rr_span(uint32_t dx0, uint32_t dx1, const ResizeRowsParams& P, uint32_t* b0, uint32_t* b1) {
    uint32_t xa, xb, t;
    float f;
    rr_axis(dx0, P.ax, P.bx, P.sw, &xa, &t, &f);
    rr_axis(dx1, P.ax, P.bx, P.sw, &t, &xb, &f);
    if (xb < xa) { const uint32_t s = xa; xa = xb; xb = s; }   // never for a >= 0; keeps the span well-formed regardless
    *b0 = (xa * 3u) & ~3u;
    *b1 = min((xb * 3u + 3u + 3u) & ~3u, P.row_floats);
}

template <int NPX, int MODE>   // MODE 1: bilinear, 2: bilinear + (v - mean) * inv_std
__global__ void __launch_bounds__(RR_THREADS) resize_rows_f32_kernel(const float* __restrict__ src, float* __restrict__ dst,
                                                                     const __grid_constant__ ResizeRowsParams P) {
    extern __shared__ __align__(128) float rr_smem[];
    __shared__ __align__(8) uint64_t full_bar[RR_MAX_STAGES];
    __shared__ __align__(8) uint64_t empty_bar[RR_MAX_STAGES];
    __shared__ float fy_s[RR_MAX_STAGES];
    constexpr uint32_t TW = RR_CT * NPX;
    constexpr uint32_t OUT_FLOATS = TW * 3u;                      // one destination row of the tile
    const uint32_t tid = threadIdx.x;
    const uint32_t nst = P.stages;
    const uint32_t stage_floats = P.slot_floats * 2u;
    float* ring = rr_smem + 2u * OUT_FLOATS;                      // [2 out rows][stages x 2 slots]
    const size_t src_img = (size_t)P.row_floats * P.sh, dst_img = (size_t)P.dw * P.dh * 3u;

    if (tid == 0) {
        for (uint32_t s = 0; s < nst; ++s) { tma::mbar_init(&full_bar[s], 1); tma::mbar_init(&empty_bar[s], RR_CT / 32); }
        tma::mbar_fence_init();
    }
    __syncthreads();

    RRWalk w;
    w.init(blockIdx.x, P);
    uint32_t stage = 0, phase = 0;

    if (tid >= RR_CT) {
        if (tid != RR_CT) return;
        // ── producer lane ──
        bool first_lap = true;
        for (uint32_t u = blockIdx.x; u < P.nunits; u += gridDim.x, w.advance(P)) {
            const uint32_t dx0 = w.tx * TW, dx1 = min(dx0 + TW, P.dw) - 1u;
            uint32_t b0, b1;
            rr_span(dx0, dx1, P, &b0, &b1);
            const uint32_t bytes = (b1 - b0) * 4u;
            const float* frame = src + (size_t)w.img * src_img + b0;
            const uint32_t y_first = w.cy * P.rows_per_chunk, y_end = min(y_first + P.rows_per_chunk, P.dh);
            for (uint32_t dy = y_first; dy < y_end; ++dy) {
                if (!first_lap) tma::mbar_wait(&empty_bar[stage], phase ^ 1u);
                uint32_t y0, y1;
                float fy;
                rr_axis(dy, P.ay, P.by, P.sh, &y0, &y1, &fy);
                float* sbase = ring + (size_t)stage * stage_floats;
                fy_s[stage] = fy;   // before the arrive(release): covered by the consumers' acquire on `full`
                tma::mbar_expect_tx(&full_bar[stage], bytes * 2u);
                tma::load_1d(sbase, frame + (size_t)y0 * P.row_floats, bytes, &full_bar[stage]);
                tma::load_1d(sbase + P.slot_floats, frame + (size_t)y1 * P.row_floats, bytes, &full_bar[stage]);
                if (++stage == nst) { stage = 0; phase ^= 1u; first_lap = false; }
            }
        }
        return;
    }

    // ── consumer warps ──
    const bool lane0 = (tid & 31u) == 0;
    uint32_t obuf = 0;
    for (uint32_t u = blockIdx.x; u < P.nunits; u += gridDim.x, w.advance(P)) {
        const uint32_t dx0 = w.tx * TW, dx1 = min(dx0 + TW, P.dw) - 1u;
        uint32_t b0, b1;
        rr_span(dx0, dx1, P, &b0, &b1);
        uint32_t o0[NPX], o1[NPX];
        float fx[NPX], gx[NPX];
#pragma unroll
        for (int j = 0; j < NPX; ++j) {
            const uint32_t x = min(dx0 + tid + (uint32_t)j * RR_CT, P.dw - 1u);   // inactive columns recompute the last one (never stored)
            uint32_t x0, x1;
            rr_axis(x, P.ax, P.bx, P.sw, &x0, &x1, &fx[j]);
            gx[j] = 1.0f - fx[j];
            o0[j] = x0 * 3u - b0;
            o1[j] = x1 * 3u - b0;
        }
        const uint32_t valid_floats = (dx1 - dx0 + 1u) * 3u;     // multiple of 4 (dw % 4 == 0, TW % 4 == 0)
        const uint32_t y_first = w.cy * P.rows_per_chunk, y_end = min(y_first + P.rows_per_chunk, P.dh);
        float* grow = dst + (size_t)w.img * dst_img + ((size_t)y_first * P.dw + dx0) * 3u;
        for (uint32_t dy = y_first; dy < y_end; ++dy) {
            tma::mbar_wait(&full_bar[stage], phase);
            const float* r0 = ring + (size_t)stage * stage_floats;
            const float* r1 = r0 + P.slot_floats;
            const float fy = fy_s[stage], gy = 1.0f - fy;
            float* orow = rr_smem + obuf * OUT_FLOATS;
#pragma unroll
            for (int j = 0; j < NPX; ++j) {
                // cuda/resize.rs:127-139 — weights first, then a left-to-right four-term sum per channel
                const float w00 = gy * gx[j], w10 = gy * fx[j], w01 = fy * gx[j], w11 = fy * fx[j];
                const float* p00 = r0 + o0[j];
                const float* p10 = r0 + o1[j];
                const float* p01 = r1 + o0[j];
                const float* p11 = r1 + o1[j];
                float c[3];
#pragma unroll
                for (int k = 0; k < 3; ++k) c[k] = w00 * p00[k] + w10 * p10[k] + w01 * p01[k] + w11 * p11[k];
                if (MODE == 2) {
                    c[0] = (c[0] - P.mean[0]) * P.inv_std[0]; c[1] = (c[1] - P.mean[1]) * P.inv_std[1]; c[2] = (c[2] - P.mean[2]) * P.inv_std[2];
                }
                float* q = orow + (tid + (uint32_t)j * RR_CT) * 3u;
                q[0] = c[0]; q[1] = c[1]; q[2] = c[2];
            }
            __syncwarp();
            if (lane0) tma::mbar_arrive(&empty_bar[stage]);
            if (++stage == nst) { stage = 0; phase ^= 1u; }
            // all four warps have written their part of the row; the other buffer is free again once everybody has passed
            // this barrier (its readers finished before they arrived here)
            tma::named_barrier(1, RR_CT);
            const float4* o4 = reinterpret_cast<const float4*>(orow);
            float4* g4 = reinterpret_cast<float4*>(grow);
#pragma unroll
            for (uint32_t k = 0; k < (OUT_FLOATS / 4u + RR_CT - 1u) / RR_CT; ++k) {
                const uint32_t v = tid + k * RR_CT;
                if (v * 4u < valid_floats) stg_stream_f4(g4 + v, o4[v]);
            }
            grow += (size_t)P.dw * 3u;
            obuf ^= 1u;
        }
    }
}

template <int NPX>
static cudaError_t rr_launch(int mode, unsigned grid, size_t smem, cudaStream_t s, const float* src, float* dst, const ResizeRowsParams& P) {
    auto go = [&](auto kern) -> cudaError_t {
        if (smem > 40 * 1024) {
            cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
            if (e != cudaSuccess) return e;
        }
        kern<<<grid, RR_THREADS, smem, s>>>(src, dst, P);
        return cudaSuccess;
    };
    return mode == 2 ? go(resize_rows_f32_kernel<NPX, 2>) : go(resize_rows_f32_kernel<NPX, 1>);
}

template <int NPX>
static int rr_occupancy(int mode, size_t smem) {
    int n = 0;
    if (smem > 40 * 1024) {   // the occupancy calculator honours the opt-in limit: raise it first
        cudaError_t a = mode == 2 ? cudaFuncSetAttribute(resize_rows_f32_kernel<NPX, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)
                                  : cudaFuncSetAttribute(resize_rows_f32_kernel<NPX, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (a != cudaSuccess) { cudaGetLastError(); return 0; }
    }
    cudaError_t e = mode == 2 ? cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, resize_rows_f32_kernel<NPX, 2>, RR_THREADS, smem)
                              : cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, resize_rows_f32_kernel<NPX, 1>, RR_THREADS, smem);
    if (e != cudaSuccess) { cudaGetLastError(); return 0; }
    return n;
}

// mode 1 bilinear / 2 bilinear+normalize.  Sets *handled when the staged kernel took the launch.
int launch_resize_rows_f32(int mode, cudaStream_t s, const float* src, float* dst, uint32_t sw, uint32_t sh, uint32_t dw, uint32_t dh,
                           uint32_t batch, float ax, float bx, float ay, float by, const float* mean, const float* inv_std, bool* handled) {
    *handled = false;
    // TMA row copies need 16-byte aligned rows; the vector stores need 16-byte aligned destination rows
    if ((sw & 3u) || (dw & 3u) || !aligned16(src) || !aligned16(dst) || sw < 8u || dw < 4u) return KB200_OK;
    if (!(ax >= 0.0f) || !(ax <= 16.0f)) return KB200_OK;   // very strong downscales: the span would be mostly unused bytes
    int npx = 1;
    {
        static const int order[3] = {2, 1, 3};
        double best = 1e30;
        for (int i = 0; i < 3; ++i) {
            const uint32_t tw = RR_CT * order[i];
            const double waste = (double)((dw + tw - 1) / tw) * tw / (double)dw;
            if (waste < best - 0.02) { best = waste; npx = order[i]; }
        }
        const int t = knob(KNOB_RS_NPX);
        if (t >= 1 && t <= 3) npx = t;
    }
    const uint32_t TW = RR_CT * (uint32_t)npx;
    ResizeRowsParams P;
    P.sw = sw; P.sh = sh; P.dw = dw; P.dh = dh;
    P.ax = ax; P.bx = bx; P.ay = ay; P.by = by;
    for (int c = 0; c < 3; ++c) { P.mean[c] = mean ? mean[c] : 0.0f; P.inv_std[c] = inv_std ? inv_std[c] : 1.0f; }
    P.row_floats = sw * 3u;
    // span bound: (TW-1)*ax source pixels between the first and the last x0, + the +1 tap, + rounding at both ends
    const double span_px = (double)(TW - 1) * (double)ax + 4.0;
    uint32_t slot = (uint32_t)(span_px * 3.0) + 8u;
    slot = (slot + 31u) & ~31u;
    slot = std::min(slot, (P.row_floats + 31u) & ~31u);
    P.slot_floats = slot;
    const size_t stage_bytes = (size_t)slot * 2u * 4u, out_bytes = (size_t)TW * 3u * 4u * 2u;
    uint32_t stages = 3;
    if (knob(KNOB_RS_STAGES) >= 2 && knob(KNOB_RS_STAGES) <= RR_MAX_STAGES) stages = (uint32_t)knob(KNOB_RS_STAGES);
    size_t smem = out_bytes + stage_bytes * stages;
    while (smem > 200 * 1024 && stages > 2) { --stages; smem = out_bytes + stage_bytes * stages; }
    if (smem > 200 * 1024) return KB200_OK;
    P.stages = stages;
    int resident = npx == 1 ? rr_occupancy<1>(mode, smem) : (npx == 2 ? rr_occupancy<2>(mode, smem) : rr_occupancy<3>(mode, smem));
    if (resident < 1) return KB200_OK;
    // ~64 KB of row copies in flight per SM covers the HBM latency; more CTAs than that only queue in the memory system
    // (knobs rs.npx / rs.stages / rs.ctas re-sweep the choice)
    int per_sm = (int)std::lround(64.0 * 1024.0 / (double)(stage_bytes * stages));
    per_sm = std::max(2, std::min(per_sm, 8));
    if (knob(KNOB_RS_CTAS) > 0) per_sm = knob(KNOB_RS_CTAS);
    per_sm = std::min(per_sm, resident);
    P.tiles_x = (dw + TW - 1) / TW;
    const size_t ctas = (size_t)device_info().sm_count * per_sm;
    const size_t total_rows = (size_t)dh * batch * P.tiles_x;
    uint32_t rc = (uint32_t)std::max<size_t>(8, total_rows / (ctas * 16));
    rc = std::min(rc, dh);
    P.rows_per_chunk = rc;
    P.chunks_y = (dh + rc - 1) / rc;
    const size_t nunits = (size_t)P.tiles_x * P.chunks_y * batch;
    if (nunits > 0x7FFFFFFFull) return KB200_OK;
    P.nunits = (uint32_t)nunits;
    const unsigned grid = (unsigned)std::min<size_t>(nunits, ctas);
    P.dtx = grid % P.tiles_x;
    const uint32_t g = grid / P.tiles_x;
    P.dcy = g % P.chunks_y;
    P.dimg = g / P.chunks_y;
    cudaError_t e = npx == 1 ? rr_launch<1>(mode, grid, smem, s, src, dst, P) : (npx == 2 ? rr_launch<2>(mode, grid, smem, s, src, dst, P) : rr_launch<3>(mode, grid, smem, s, src, dst, P));
    if (e != cudaSuccess) return fail(KB200_ERR_CUDA, "cudaFuncSetAttribute failed: %s", cudaGetErrorString(e));
    KB200_TRY(check_launch("resize_rows_f32_kernel"));
    *handled = true;
    return KB200_OK;
}

}  // namespace kb200
