// normalize.cu — normalize_mean_std / normalize_rgb_u8 / find_min_max / normalize_min_max (a10)
// and std_mean (a11).
//
// Reference: normalize.rs:56-87, :123-146, :191-222, :235-263 (+ scalar leaf :407-421, AVX2 leaf with
// fmadd on the npixels&~7 bulk), core.rs:42-67.
//
// Design: streaming kernels over flat arrays with lane-contiguous 16-byte vector accesses in both
// directions (the channel phase of a vector is (index % 3), loop-invariant per thread); reductions use
// per-thread integer accumulators, warp shuffles and one atomic per CTA, so `std_mean`'s sums are
// exact integers independent of the order of accumulation (= the reference's f64 folds, which are
// exact below 2^53).
#include <algorithm>

#include "kb200_common.cuh"

namespace kb200 {

struct Ch4 { float v[4]; };

// (x - mean[c]) / std[c] — IEEE division (normalize.rs:76-84).
// Flat float4 indexing: lane i of a warp touches bytes [16i, 16i+16) of a 512-B run, so every LDG.128 / STG.128 is
// lane-contiguous (a first version gave each thread 3 consecutive float4 = 48-B lane stride: every store
// instruction then half-filled its sectors — same defect ncu showed on the NV12 kernel).  Element e = 4q + j is
// channel (q + j) % 3; the grid stride is a multiple of 3 so a thread's channel phase is loop-invariant.
__global__ void __launch_bounds__(256) normalize_mean_std_c3_vec(const float4* __restrict__ src, float4* __restrict__ dst,
                                                                 size_t nvec, Ch4 mean, Ch4 stdv) {
    const size_t stride = (size_t)gridDim.x * blockDim.x;  // multiple of 3 (launcher)
    size_t q = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t ph = (uint32_t)(q % 3);
    const float m[3] = {mean.v[0], mean.v[1], mean.v[2]}, sd[3] = {stdv.v[0], stdv.v[1], stdv.v[2]};
    const float ma = ph == 0 ? m[0] : (ph == 1 ? m[1] : m[2]), mb = ph == 0 ? m[1] : (ph == 1 ? m[2] : m[0]),
                mc = ph == 0 ? m[2] : (ph == 1 ? m[0] : m[1]);
    const float sa = ph == 0 ? sd[0] : (ph == 1 ? sd[1] : sd[2]), sb = ph == 0 ? sd[1] : (ph == 1 ? sd[2] : sd[0]),
                sc = ph == 0 ? sd[2] : (ph == 1 ? sd[0] : sd[1]);
    auto norm4 = [&](float4 v) {
        v.x = __fdiv_rn(v.x - ma, sa); v.y = __fdiv_rn(v.y - mb, sb); v.z = __fdiv_rn(v.z - mc, sc); v.w = __fdiv_rn(v.w - ma, sa);
        return v;
    };
    // four independent 16-B loads in flight per thread: ncu on the one-load loop showed full occupancy, low issue and
    // long-scoreboard stalls — one 16-B load per thread in flight per SM is short of bandwidth x latency
    for (; q + 3 * stride < nvec; q += 4 * stride) {
        const float4 a = ldg_stream_f4(src + q), b = ldg_stream_f4(src + q + stride), c = ldg_stream_f4(src + q + 2 * stride),
                     d = ldg_stream_f4(src + q + 3 * stride);
        stg_stream_f4(dst + q, norm4(a)); stg_stream_f4(dst + q + stride, norm4(b));
        stg_stream_f4(dst + q + 2 * stride, norm4(c)); stg_stream_f4(dst + q + 3 * stride, norm4(d));
    }
    for (; q < nvec; q += stride) stg_stream_f4(dst + q, norm4(ldg_stream_f4(src + q)));
}

__global__ void normalize_mean_std_generic(const float* __restrict__ src, float* __restrict__ dst, size_t first, size_t n,
                                           uint32_t C, Ch4 mean, Ch4 stdv) {
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (size_t i = first + (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const uint32_t c = (uint32_t)(i % C);
        dst[i] = __fdiv_rn(__ldg(src + i) - mean.v[c], stdv.v[c]);
    }
}

// u8*scale[c] + offset[c]; FMA for pixels < bulk (AVX2/NEON leaves), mul+add otherwise.
__device__ __forceinline__ float norm_u8(float v, float sc, float of, bool fused) { return fused ? fmaf(v, sc, of) : v * sc + of; }

// One 32-bit word in (4 bytes), one STG.128 out per thread-iteration: both lane-contiguous.  Byte j of word q is
// element 4q + j = channel (q + j) % 3; grid stride is a multiple of 3.
__global__ void __launch_bounds__(256) normalize_rgb_u8_vec(const uint32_t* __restrict__ src, float4* __restrict__ dst,
                                                            size_t nwords, Ch4 scale, Ch4 offset, size_t bulk_elems) {
    const size_t stride = (size_t)gridDim.x * blockDim.x;  // multiple of 3 (launcher)
    size_t q = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t ph = (uint32_t)(q % 3);
    const float s[3] = {scale.v[0], scale.v[1], scale.v[2]}, o[3] = {offset.v[0], offset.v[1], offset.v[2]};
    const float sa = ph == 0 ? s[0] : (ph == 1 ? s[1] : s[2]), sb = ph == 0 ? s[1] : (ph == 1 ? s[2] : s[0]),
                sc = ph == 0 ? s[2] : (ph == 1 ? s[0] : s[1]);
    const float oa = ph == 0 ? o[0] : (ph == 1 ? o[1] : o[2]), ob = ph == 0 ? o[1] : (ph == 1 ? o[2] : o[0]),
                oc = ph == 0 ? o[2] : (ph == 1 ? o[0] : o[1]);
    auto norm4 = [&](uint32_t w, size_t qq) {
        const bool f = 4 * qq < bulk_elems;  // bulk = 8-px multiple = 24-element multiple: a word never straddles it
        float4 v;
        v.x = norm_u8(byte_to_float(w, 0), sa, oa, f); v.y = norm_u8(byte_to_float(w, 1), sb, ob, f);
        v.z = norm_u8(byte_to_float(w, 2), sc, oc, f); v.w = norm_u8(byte_to_float(w, 3), sa, oa, f);
        return v;
    };
    for (; q + 3 * stride < nwords; q += 4 * stride) {   // four loads in flight per thread (see normalize_mean_std_c3_vec)
        const uint32_t a = __ldg(src + q), b = __ldg(src + q + stride), c = __ldg(src + q + 2 * stride), d = __ldg(src + q + 3 * stride);
        stg_stream_f4(dst + q, norm4(a, q)); stg_stream_f4(dst + q + stride, norm4(b, q + stride));
        stg_stream_f4(dst + q + 2 * stride, norm4(c, q + 2 * stride)); stg_stream_f4(dst + q + 3 * stride, norm4(d, q + 3 * stride));
    }
    for (; q < nwords; q += stride) stg_stream_f4(dst + q, norm4(__ldg(src + q), q));
}

__global__ void normalize_rgb_u8_generic(const uint8_t* __restrict__ src, float* __restrict__ dst, size_t first_px,
                                         size_t npixels, Ch4 scale, Ch4 offset, size_t bulk_px) {
    const size_t i = first_px + (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= npixels) return;
    const bool f = i < bulk_px;
#pragma unroll
    for (int c = 0; c < 3; ++c) dst[3 * i + c] = norm_u8((float)src[3 * i + c], scale.v[c], offset.v[c], f);
}

// ── min / max ───────────────────────────────────────────────────────────────────────────────
// Order-preserving float <-> uint32 map so atomicMin/atomicMax on integers implement float min/max.
__device__ __forceinline__ uint32_t f2ord(float f) {
    const uint32_t u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float ord2f(uint32_t o) {
    const uint32_t u = (o & 0x80000000u) ? (o & 0x7FFFFFFFu) : ~o;
    return __uint_as_float(u);
}

__global__ void minmax_init_kernel(uint32_t* mm) { mm[0] = 0xFFFFFFFFu; mm[1] = 0u; }

// find_min_max (normalize.rs:123-146): strict `<` / `>` scans from the first element — the result is
// the minimum / maximum under IEEE ordering; NaNs never win a comparison (same here: fminf/fmaxf-free,
// comparisons only).
__global__ void __launch_bounds__(256) minmax_kernel(const float* __restrict__ src, size_t n, uint32_t* mm) {
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    float lo = __int_as_float(0x7F800000), hi = __int_as_float(0xFF800000);
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const float v = __ldg(src + i);
        if (v < lo) lo = v;
        if (v > hi) hi = v;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float l2 = __shfl_xor_sync(0xFFFFFFFFu, lo, o), h2 = __shfl_xor_sync(0xFFFFFFFFu, hi, o);
        if (l2 < lo) lo = l2;
        if (h2 > hi) hi = h2;
    }
    if ((threadIdx.x & 31) == 0) {
        atomicMin(mm, f2ord(lo));
        atomicMax(mm + 1, f2ord(hi));
    }
}

// The reference seeds min and max with the FIRST element (normalize.rs:128-134): a NaN first element never loses a
// comparison, so the result is (NaN, NaN) — reproduced here.  NaNs elsewhere never win (same as the reference).
// Ties between -0.0 and +0.0 resolve to -0.0 for min / +0.0 for max (bit-pattern order) instead of first occurrence;
// the two are numerically equal and normalize_min_max differs only in the sign of an exact zero.
__global__ void minmax_finish_kernel(uint32_t* mm, const float* __restrict__ src) {
    float* f = reinterpret_cast<float*>(mm);
    const float first = src[0];
    float lo = ord2f(mm[0]), hi = ord2f(mm[1]);
    if (first != first) { lo = first; hi = first; }
    f[0] = lo; f[1] = hi;
}

// (x - min_val) * (max - min) / (max_val - min_val) + min   (normalize.rs:213-218)
__global__ void __launch_bounds__(256) normalize_min_max_kernel(const float* __restrict__ src, float* __restrict__ dst,
                                                                size_t n, float mn, float mx,
                                                                const float* __restrict__ minmax) {
    const float min_val = minmax[0], max_val = minmax[1];
    const float range = mx - mn, denom = max_val - min_val;
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
        dst[i] = __fdiv_rn((__ldg(src + i) - min_val) * range, denom) + mn;
}

// ── std_mean ────────────────────────────────────────────────────────────────────────────────
// Flat u8 stream read as lane-contiguous 16-byte vectors (LDG.128: 512 contiguous bytes per warp).  Byte j of
// vector q is element 16q + j = channel (q + j) % 3; the grid stride is a multiple of 3, so a thread accumulates
// into three phase-RELATIVE accumulators and rotates them to absolute channels once at the end.  Per-thread u32
// accumulators are flushed into u64 before they can overflow (255² * 6 bytes * 8192 vectors < 2^32).
// `head` = leading bytes (0..15) in front of the first 16-byte-aligned address: they and the tail are summed byte-wise
// by one thread; the vector body starts at src + head, which rotates the channel phase by head % 3.
__global__ void __launch_bounds__(256) std_mean_kernel(const uint8_t* __restrict__ src, size_t nbytes, uint32_t head, size_t nvec,
                                                       unsigned long long* __restrict__ sums) {
    unsigned long long s64[3] = {0, 0, 0}, q64[3] = {0, 0, 0};  // phase-relative
    uint32_t s32[3] = {0, 0, 0}, q32[3] = {0, 0, 0};
    const size_t stride = (size_t)gridDim.x * blockDim.x;  // multiple of 3 (launcher)
    size_t q = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t ph = (uint32_t)((q + head) % 3);
    uint32_t pending = 0;
    const uint4* v4 = reinterpret_cast<const uint4*>(src + head);
    // byte j of word kk is relative channel (kk + j) % 3.  DP4A does the byte sums: Σ b·sel for the plain sums,
    // Σ b·(b & mask) for the squares — 3 LOP + 6 IDP4A per word instead of ~20 scalar ops.
    auto accumulate = [&](const uint4& v) {
        const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
            for (int r = 0; r < 3; ++r) {
                uint32_t sel = 0, mask = 0;
#pragma unroll
                for (int j = 0; j < 4; ++j)
                    if ((kk + j) % 3 == r) { sel |= 1u << (8 * j); mask |= 0xFFu << (8 * j); }
                s32[r] = __dp4a(w[kk], sel, s32[r]);
                q32[r] = __dp4a(w[kk], w[kk] & mask, q32[r]);
            }
        }
    };
    auto flush = [&]() {
#pragma unroll
        for (int c = 0; c < 3; ++c) { s64[c] += s32[c]; q64[c] += q32[c]; s32[c] = 0; q32[c] = 0; }
        pending = 0;
    };
    // four independent 16-B loads in flight per thread (the one-load loop is latency-bound, see normalize_mean_std_c3_vec);
    // the stride is a multiple of 3, so all four vectors share the thread's channel phase
    for (; q + 3 * stride < nvec; q += 4 * stride) {
        const uint4 a = ldg_stream_u4(v4 + q), b = ldg_stream_u4(v4 + q + stride), c = ldg_stream_u4(v4 + q + 2 * stride),
                    d = ldg_stream_u4(v4 + q + 3 * stride);
        accumulate(a); accumulate(b); accumulate(c); accumulate(d);
        pending += 4;
        if (pending >= 8192u) flush();   // 255^2 * 6 bytes * 8192 vectors < 2^32
    }
    for (; q < nvec; q += stride) {
        accumulate(ldg_stream_u4(v4 + q));
        if (++pending >= 8192u) flush();
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) { s64[c] += s32[c]; q64[c] += q32[c]; }
    // rotate relative -> absolute: relative slot r holds channel (ph + r) % 3
    unsigned long long sa[3], qa[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const uint32_t r = (c + 3u - ph) % 3u;  // slot holding channel c
        sa[c] = r == 0 ? s64[0] : (r == 1 ? s64[1] : s64[2]);
        qa[c] = r == 0 ? q64[0] : (r == 1 ? q64[1] : q64[2]);
    }
    // head (< 16) and tail (< 16) bytes — thread 0 of CTA 0
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        auto add_byte = [&](size_t e) {
            const uint32_t b = src[e];
            const uint32_t c = (uint32_t)(e % 3);
            if (c == 0) { sa[0] += b; qa[0] += b * b; } else if (c == 1) { sa[1] += b; qa[1] += b * b; } else { sa[2] += b; qa[2] += b * b; }
        };
        for (size_t e = 0; e < head && e < nbytes; ++e) add_byte(e);
        for (size_t e = (size_t)head + nvec * 16; e < nbytes; ++e) add_byte(e);
    }
    __shared__ unsigned long long red[6][8];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            sa[c] += __shfl_xor_sync(0xFFFFFFFFu, sa[c], o);
            qa[c] += __shfl_xor_sync(0xFFFFFFFFu, qa[c], o);
        }
    }
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0) {
#pragma unroll
        for (int c = 0; c < 3; ++c) { red[c][warp] = sa[c]; red[3 + c][warp] = qa[c]; }
    }
    __syncthreads();
    if (threadIdx.x < 6) {
        unsigned long long t = 0;
        for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += red[threadIdx.x][w];
        atomicAdd(sums + threadIdx.x, t);
    }
}

// grid whose total thread count is a multiple of 3 (block = 256 ⇒ grid multiple of 3)
static inline unsigned stream_grid3(size_t items, unsigned block, unsigned ctas_per_sm) {
    const size_t want = (items + block - 1) / block;
    const size_t cap = (size_t)device_info().sm_count * ctas_per_sm;
    size_t g = std::max<size_t>(1, std::min(want, cap));
    g = (g + 2) / 3 * 3;
    return (unsigned)g;
}

static inline unsigned stream_grid(size_t items, unsigned block, unsigned ctas_per_sm) {
    const size_t want = (items + block - 1) / block;
    const size_t cap = (size_t)device_info().sm_count * ctas_per_sm;
    return (unsigned)std::max<size_t>(1, std::min(want, cap));
}

}  // namespace kb200

using namespace kb200;

extern "C" {

KB200_API int kb200_normalize_mean_std_f32(kb200_stream_t stream, const float* src, float* dst, size_t npixels,
                                           uint32_t channels, const float* mean, const float* stdv) {
    KB200_TRY(check_ptr("src", src)); KB200_TRY(check_ptr("dst", dst));
    KB200_TRY(check_ptr("mean", mean)); KB200_TRY(check_ptr("std", stdv));
    if (channels == 0 || channels > 4) return fail(KB200_ERR_UNSUPPORTED, "normalize_mean_std supports 1..4 channels, got %u", channels);
    if (npixels == 0) return KB200_OK;
    Ch4 m{}, sd{};
    for (uint32_t c = 0; c < channels; ++c) { m.v[c] = mean[c]; sd.v[c] = stdv[c]; }
    cudaStream_t s = as_stream(stream);
    const size_t n = npixels * channels;
    size_t done = 0;
    if (channels == 3 && aligned16(src) && aligned16(dst)) {
        const size_t nvec = n / 4;
        if (nvec) {
            normalize_mean_std_c3_vec<<<stream_grid3(nvec, 256, 8), 256, 0, s>>>(
                reinterpret_cast<const float4*>(src), reinterpret_cast<float4*>(dst), nvec, m, sd);
            KB200_TRY(check_launch("normalize_mean_std_c3_vec"));
        }
        done = nvec * 4;
    }
    if (done < n) {
        normalize_mean_std_generic<<<stream_grid(n - done, 256, 8), 256, 0, s>>>(src, dst, done, n, channels, m, sd);
        KB200_TRY(check_launch("normalize_mean_std_generic"));
    }
    return KB200_OK;
}

KB200_API int kb200_normalize_rgb_u8_f32(kb200_stream_t stream, const uint8_t* src, float* dst, size_t npixels,
                                         const float scale[3], const float offset[3], int leaf) {
    KB200_TRY(check_ptr("src", src)); KB200_TRY(check_ptr("dst", dst));
    KB200_TRY(check_ptr("scale", scale)); KB200_TRY(check_ptr("offset", offset));
    if (leaf < 0 || leaf > 2) return fail(KB200_ERR_INVALID_ARGUMENT, "unknown cpu leaf %d", leaf);
    if (npixels == 0) return KB200_OK;
    Ch4 sc{}, of{};
    for (int c = 0; c < 3; ++c) { sc.v[c] = scale[c]; of.v[c] = offset[c]; }
    const size_t bulk = (leaf == KB200_LEAF_SCALAR) ? 0 : (npixels & ~(size_t)7);
    cudaStream_t s = as_stream(stream);
    size_t done = 0;
    if (aligned4(src) && aligned16(dst)) {
        const size_t nwords = npixels * 3 / 4;
        if (nwords) {
            normalize_rgb_u8_vec<<<stream_grid3(nwords, 256, 8), 256, 0, s>>>(
                reinterpret_cast<const uint32_t*>(src), reinterpret_cast<float4*>(dst), nwords, sc, of, bulk * 3);
            KB200_TRY(check_launch("normalize_rgb_u8_vec"));
        }
        done = nwords * 4 / 3;  // whole pixels covered by the vector pass
    }
    if (done < npixels) {
        normalize_rgb_u8_generic<<<div_up(npixels - done, 256), 256, 0, s>>>(src, dst, done, npixels, sc, of, bulk);
        KB200_TRY(check_launch("normalize_rgb_u8_generic"));
    }
    return KB200_OK;
}

KB200_API int kb200_find_min_max_f32(kb200_stream_t stream, const float* src, size_t n, float* minmax_dev) {
    KB200_TRY(check_ptr("src", src)); KB200_TRY(check_ptr("minmax_dev", minmax_dev));
    if (n == 0) return fail(KB200_ERR_INVALID_ARGUMENT, "image data is not initialized (empty image)");  // ImageDataNotInitialized
    cudaStream_t s = as_stream(stream);
    uint32_t* mm = reinterpret_cast<uint32_t*>(minmax_dev);
    minmax_init_kernel<<<1, 1, 0, s>>>(mm);
    minmax_kernel<<<stream_grid(n, 256, 8), 256, 0, s>>>(src, n, mm);
    minmax_finish_kernel<<<1, 1, 0, s>>>(mm, src);
    return check_launch("minmax_kernel");
}

KB200_API int kb200_normalize_min_max_f32(kb200_stream_t stream, const float* src, float* dst, size_t n, float mn,
                                          float mx, const float* minmax_dev) {
    KB200_TRY(check_ptr("src", src)); KB200_TRY(check_ptr("dst", dst)); KB200_TRY(check_ptr("minmax_dev", minmax_dev));
    if (n == 0) return fail(KB200_ERR_INVALID_ARGUMENT, "image data is not initialized (empty image)");
    normalize_min_max_kernel<<<stream_grid(n, 256, 8), 256, 0, as_stream(stream)>>>(src, dst, n, mn, mx, minmax_dev);
    return check_launch("normalize_min_max_kernel");
}

KB200_API int kb200_std_mean_u8_c3(kb200_stream_t stream, const uint8_t* src, size_t npixels, uint64_t* sums_dev) {
    KB200_TRY(check_ptr("src", src)); KB200_TRY(check_ptr("sums_dev", sums_dev));
    cudaStream_t s = as_stream(stream);
    cudaError_t e = cudaMemsetAsync(sums_dev, 0, 6 * sizeof(uint64_t), s);
    if (e != cudaSuccess) return fail(KB200_ERR_CUDA, "cudaMemsetAsync failed: %s", cudaGetErrorString(e));
    if (npixels == 0) return KB200_OK;
    const size_t nbytes = npixels * 3;
    // an unaligned base (a tensor slice) peels up to 15 leading bytes; the vector body then runs on the aligned remainder
    const uint32_t head = (uint32_t)((16u - (uint32_t)(reinterpret_cast<uintptr_t>(src) & 15u)) & 15u);
    const size_t nvec = nbytes > head ? (nbytes - head) / 16 : 0;
    std_mean_kernel<<<stream_grid3(std::max<size_t>(nvec, 1), 256, 6), 256, 0, s>>>(src, nbytes, head, nvec, reinterpret_cast<unsigned long long*>(sums_dev));
    return check_launch("std_mean_kernel");
}

}  // extern "C"
