// filter.cu — separable f32 filters: separable_filter, gaussian_blur, sobel (a6, a7; config 4).
//
// Reference: filter/separable_filter.rs:87-155 (CPU engine: H pass into a full f32 `temp` image,
// then V pass; correlation; taps ascending; `acc += v * k` unfused; out-of-bounds taps SKIPPED =
// constant-zero border, no renormalisation), filter/ops.rs:116-203 (gaussian_blur, sobel),
// cuda/filter.rs:55-110, :515-565 and filter/cuda.rs:106-232 (GPU twin: 2 launches through a DRAM
// scratch image for a blur, 5 launches / 11 image traversals for sobel).
//
// Design: ONE kernel per op.  A CTA stages a (TH + ky-1) x (TW + kx-1) pixel tile (zero-filled
// outside the image) in shared memory, runs the H pass into a second shared tile and the V pass
// straight to global memory — the f32 intermediate never touches HBM (traffic: 1 read + 1 write of
// the image instead of 2+2; sobel: 1+1 instead of 11).  Sobel runs both gradient filters off the
// same staged tile and fuses the magnitude.
//
// Bit-exactness with the two-pass reference: each intermediate value is the same ascending,
// unfused (-fmad=false) accumulation starting from +0.0.  A zero-filled halo element contributes
// `acc += 0*k` = acc (acc can never be -0.0: it starts at +0.0 and x + (-x) rounds to +0.0), which
// equals "tap skipped" for every finite tap.  (Non-finite taps × zero halo would differ; taps come
// from finite Gaussian/Sobel tables.)
#include <algorithm>

#include <cstdio>
#include <cstdlib>
#include <type_traits>

#include "kb200_common.cuh"
#include "pair_math.cuh"

namespace kb200 {

static constexpr int KB200_MAX_TAPS = 31;

struct SepTaps {
    float kx[32];
    float ky[32];
    int kxn, kyn;
};

struct SepGeom {
    uint32_t cols, rows, C;
    uint32_t tw, th;          // tile size in pixels
    uint32_t tiles_x, tiles_y;
};

// KX/KY > 0: compile-time tap counts (fully unrolled); 0: runtime loops.
// SOBEL: kx = derivative taps, ky = smoothing taps (same length); gx = H(kx)·V(ky), gy = H(ky)·V(kx),
// out = sqrt(gx*gx + gy*gy)   (filter/ops.rs:187-200)
template <int KX, int KY, bool SOBEL>
__global__ void __launch_bounds__(256) sep_filter_fused_kernel(const float* __restrict__ src, float* __restrict__ dst,
                                                               const __grid_constant__ SepTaps taps,
                                                               const __grid_constant__ SepGeom g) {
    extern __shared__ __align__(16) float smem[];
    const int kxn = KX > 0 ? KX : taps.kxn, kyn = KY > 0 ? KY : taps.kyn;
    const int hx = kxn / 2, hy = kyn / 2;  // offsets_x = i - half  (separable_filter.rs:60-69)
    const int C = (int)g.C;
    const int in_w = ((int)g.tw + kxn - 1) * C;  // floats per staged row
    const int mid_w = (int)g.tw * C;
    const int in_h = (int)g.th + kyn - 1;
    float* s_in = smem;
    float* s_mid = smem + (size_t)in_w * in_h;             // [in_h][mid_w]
    float* s_mid2 = SOBEL ? s_mid + (size_t)mid_w * in_h : nullptr;

    const uint32_t tile = blockIdx.x;
    const uint32_t tx = tile % g.tiles_x, ty = (tile / g.tiles_x) % g.tiles_y, img = tile / (g.tiles_x * g.tiles_y);
    const int x0 = (int)(tx * g.tw), y0 = (int)(ty * g.th);
    const size_t img_off = (size_t)img * g.cols * g.rows * C;
    const float* s = src + img_off;
    const int row_floats = (int)g.cols * C;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;

    // phase 1: stage the input tile, zero outside the image
    const int gx_base = (x0 - hx) * C;
    for (int r = warp; r < in_h; r += nwarps) {
        const int gy = y0 - hy + r;
        const bool row_ok = gy >= 0 && gy < (int)g.rows;
        const float* grow = s + (size_t)(row_ok ? gy : 0) * row_floats;
        float* srow = s_in + (size_t)r * in_w;
        for (int j = lane; j < in_w; j += 32) {
            const int gxf = gx_base + j;
            srow[j] = (row_ok && gxf >= 0 && gxf < row_floats) ? __ldg(grow + gxf) : 0.0f;
        }
    }
    __syncthreads();

    // phase 2: horizontal pass  temp[r][e] = Σ_t in[r][e + t*C] * kx[t]
    for (int r = warp; r < in_h; r += nwarps) {
        const float* srow = s_in + (size_t)r * in_w;
        for (int e = lane; e < mid_w; e += 32) {
            float acc = 0.0f, acc2 = 0.0f;
            if (KX > 0) {
#pragma unroll
                for (int t = 0; t < (KX > 0 ? KX : 1); ++t) {
                    const float v = srow[e + t * C];
                    acc += v * taps.kx[t];
                    if (SOBEL) acc2 += v * taps.ky[t];
                }
            } else {
                for (int t = 0; t < kxn; ++t) {
                    const float v = srow[e + t * C];
                    acc += v * taps.kx[t];
                    if (SOBEL) acc2 += v * taps.ky[t];
                }
            }
            s_mid[(size_t)r * mid_w + e] = acc;
            if (SOBEL) s_mid2[(size_t)r * mid_w + e] = acc2;
        }
    }
    __syncthreads();

    // phase 3: vertical pass straight to global memory
    const int out_w = min((int)g.tw, (int)g.cols - x0) * C;
    float* d = dst + img_off;
    for (int r = warp; r < (int)g.th; r += nwarps) {
        const int gy = y0 + r;
        if (gy >= (int)g.rows) break;
        float* drow = d + (size_t)gy * row_floats + (size_t)x0 * C;
        for (int e = lane; e < out_w; e += 32) {
            float acc = 0.0f, acc2 = 0.0f;
            if (KY > 0) {
#pragma unroll
                for (int t = 0; t < (KY > 0 ? KY : 1); ++t) {
                    acc += s_mid[(size_t)(r + t) * mid_w + e] * taps.ky[t];
                    if (SOBEL) acc2 += s_mid2[(size_t)(r + t) * mid_w + e] * taps.kx[t];
                }
            } else {
                for (int t = 0; t < kyn; ++t) {
                    acc += s_mid[(size_t)(r + t) * mid_w + e] * taps.ky[t];
                    if (SOBEL) acc2 += s_mid2[(size_t)(r + t) * mid_w + e] * taps.kx[t];
                }
            }
            drow[e] = SOBEL ? sqrtf(acc * acc + acc2 * acc2) : acc;
        }
    }
}

// ─────────────────────────────────────────────────────────────────────────────────────────────
// Row-streaming kernel (the config-4 fast path): C ∈ {1,3,4}, taps ∈ {3,5,7}, (cols*C) % 4 == 0.
//
// ncu on the tile kernel above: K LDS + 2K FP per pass per element plus 64-bit index math in the tap loops —
// issue-bound, far below the HBM roofline.  Here:
//   * work unit = (image, strip of 512*NV floats of a row, chunk of `rows_per_chunk` rows); a CTA walks its
//     strip top-down.  Each input row segment (strip + 16-B-rounded halo) is copied global -> shared by
//     the TMA engine (cp.async.bulk 1-D) into an mbarrier ring by a producer warp — every input row is
//     read once per chunk (+ K-1 halo rows per chunk), nothing is staged twice horizontally.
//   * a consumer thread owns NV float4 columns of the strip (tid, tid+128, …; each lane-contiguous).  Per row it
//     reads its outputs' horizontal support as NF4 aligned LDS.128, forms the horizontal results in registers,
//     pushes them into a K-deep register window (rotation is free: the row loop is unrolled K times) and emits
//     the vertical result of the row that just became complete with lane-contiguous STG.128.
//   * the f32 intermediate never leaves the register file.
// Zero border: rows outside the image are not copied — the producer just arrives and flags the row, the
// consumer pushes zeros; float4s left/right of the image row are zeroed in registers (edge strips only; interior
// strips run a copy of the row loop with no bounds logic).
// Arithmetic per output is the reference's: acc = 0; acc += v*k in ascending tap order, unfused.

struct SepStreamParams {
    uint32_t rowlen;       // cols * C floats
    uint32_t rows, batch;
    uint32_t strips, chunks, rows_per_chunk, nunits;
    uint32_t slot_floats;  // floats per stage slot
};

__device__ __forceinline__ uint32_t ss_smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void ss_mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(ss_smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void ss_mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(ss_smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void ss_mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(ss_smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void ss_mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "SS_WAIT_LOOP:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra SS_WAIT_DONE;\n"
        "bra SS_WAIT_LOOP;\n"
        "SS_WAIT_DONE:\n"
        "}\n" ::"r"(ss_smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void ss_tma_load_1d(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(ss_smem_u32(smem_dst)),
                 "l"(gmem_src), "r"(bytes), "r"(ss_smem_u32(bar))
                 : "memory");
}

// Sobel taps are compile-time constants (filter/kernels.rs:55-72): D = derivative, S = smoothing.
template <int K> struct SobelTaps;
template <> struct SobelTaps<3> { static constexpr int D[3] = {-1, 0, 1}; static constexpr int S[3] = {1, 2, 1}; };
template <> struct SobelTaps<5> { static constexpr int D[5] = {-1, -2, 0, 2, 1}; static constexpr int S[5] = {1, 4, 6, 4, 1}; };

// acc + v*k for a compile-time integer tap, bit-identical to the reference's unfused `acc += v * k`:
//   k == 0      : v*0 = ±0 and acc + ±0 = acc (acc is never -0: every accumulation starts from +0.0) — skipped;
//   |k| = 2^n   : the product is exact, so one FFMA (single rounding of acc + v*k) equals mul-then-add;
//   otherwise   : mul, then add.
// (Finite inputs, like the zero-halo argument in the file header.)
template <int KV>
__device__ __forceinline__ float acc_tap(float acc, float v) {
    if (KV == 0) return acc;
    if (KV == 1) return acc + v;
    if (KV == -1) return acc - v;
    if ((KV & (KV - 1)) == 0 || ((-KV) & (-KV - 1)) == 0) return fmaf(v, (float)KV, acc);
    return acc + v * (float)KV;
}
template <int K, bool DERIV, int T>
struct SobelAcc {
    template <typename F>
    __device__ __forceinline__ static float run(float acc, F&& get) {
        constexpr int kv = DERIV ? SobelTaps<K>::D[T] : SobelTaps<K>::S[T];
        acc = acc_tap<kv>(acc, kv == 0 ? 0.0f : get(T));
        if constexpr (T + 1 < K) return SobelAcc<K, DERIV, T + 1>::run(acc, get);
        else return acc;
    }
};

// ─────────────────────────────────────────────────────────────────────────────────────────────
// Paired vertical pass.
//
// ncu history: the first streaming kernel (one float4 per thread, scalar mul+add in both passes, bounds selects in
// every row) was issue-bound — unfused FMUL/FADD and mbarrier spin took most of the issue slots.
//   * the vertical pass runs on register PAIRS (fma2_rn, kb200_common.cuh: one scalar FFMA per lane on sm_90).  The
//     reference's unfused `acc += v * k` is kept bit-for-bit: the product is formed as fma2(v, k, -0) and the sum as
//     fma2(p, 1, acc) with -0 and 1 passed as kernel arguments (opaque to the optimiser), each rounding once, = mul
//     then add;
//   * the first tap of every accumulation is a single fma(v, k, +0) (== round(v*k) + 0, signed zeros included);
//   * the horizontal pass stays scalar: with C = 3 the tap pairs of neighbouring outputs alternate between even
//     and odd register offsets, and an unaligned pair costs more moves than the packed op saves;
//   * NV = 1 is what ships: two columns per thread (NV = 2) halve the per-row bookkeeping but need 77-93 registers,
//     which caps the SM at 4 CTAs / 20 warps.
template <int NV> struct SS2 {
    static constexpr int COLS4 = 128;               // consumer threads
    static constexpr int EW = COLS4 * 4 * NV;       // floats per strip
    static constexpr int THREADS = COLS4 + 32;
    static constexpr int MAX_STAGES = 12;
};

typedef unsigned long long ss_u64;
__device__ __forceinline__ ss_u64 ss_pack(float a, float b) { ss_u64 r; asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(a), "f"(b)); return r; }
__device__ __forceinline__ void ss_unpack(ss_u64 v, float& a, float& b) { asm("mov.b64 {%0, %1}, %2;" : "=f"(a), "=f"(b) : "l"(v)); }
__device__ __forceinline__ ss_u64 ss_fma2(ss_u64 a, ss_u64 b, ss_u64 c) { return fma2_rn(a, b, c); }

// exact two-rounding helpers on pairs (see header): NZ = (-0,-0), ONE = (1,1), both opaque run-time values
struct PairConst { ss_u64 nz, one, zero; };
__device__ __forceinline__ ss_u64 pair_mul(ss_u64 v, ss_u64 k, const PairConst& c) { return ss_fma2(v, k, c.nz); }
__device__ __forceinline__ ss_u64 pair_add(ss_u64 a, ss_u64 b, const PairConst& c) { return ss_fma2(b, c.one, a); }

// acc + v*k on pairs for a compile-time integer tap (same case analysis as acc_tap above)
template <int KV>
__device__ __forceinline__ ss_u64 pair_acc_tap(ss_u64 acc, ss_u64 v, const PairConst& c) {
    if (KV == 0) return acc;
    if ((KV & (KV - 1)) == 0 || ((-KV) & (-KV - 1)) == 0) return ss_fma2(v, ss_pack((float)KV, (float)KV), acc);  // exact product: one rounding == two
    return pair_add(acc, pair_mul(v, ss_pack((float)KV, (float)KV), c), c);
}
template <int K, bool DERIV, int T>
struct SobelAccPair {
    template <typename F>
    __device__ __forceinline__ static ss_u64 run(ss_u64 acc, const PairConst& c, F&& get) {
        constexpr int kv = DERIV ? SobelTaps<K>::D[T] : SobelTaps<K>::S[T];
        if constexpr (kv != 0) acc = pair_acc_tap<kv>(acc, get(T), c);
        if constexpr (T + 1 < K) return SobelAccPair<K, DERIV, T + 1>::run(acc, c, get);
        else return acc;
    }
};

struct SepStream2Params {
    SepStreamParams g;
    uint32_t stages;
    float neg_zero, one;   // -0.0f and 1.0f, passed at run time on purpose (see header)
};

template <int C, int KX, int KY, bool SOBEL, int NV>
__global__ void __launch_bounds__(SS2<NV>::THREADS) sep_filter_stream2_kernel(const float* __restrict__ src, float* __restrict__ dst,
                                                                              const __grid_constant__ SepTaps taps,
                                                                              const __grid_constant__ SepStream2Params R) {
    using G = SS2<NV>;
    constexpr int HX = KX / 2, HY = KY / 2;
    constexpr int HL = ((HX * C + 3) / 4) * 4;                 // left halo, floats, 16-B rounded
    constexpr int HR = (((KX - 1 - HX) * C + 3) / 4) * 4;      // right halo
    constexpr int NF4 = 1 + HL / 4 + HR / 4;                   // float4s a thread reads per row per column
    constexpr int OFF = HL - HX * C;                           // in[] index of tap 0 of output 0
    extern __shared__ __align__(128) float ss_smem[];
    __shared__ __align__(8) uint64_t full_bar[G::MAX_STAGES];
    __shared__ __align__(8) uint64_t empty_bar[G::MAX_STAGES];
    __shared__ int row_valid[G::MAX_STAGES];
    const SepStreamParams& P = R.g;
    const uint32_t tid = threadIdx.x;
    const uint32_t nst = R.stages;
    if (tid == 0) {
        for (uint32_t s = 0; s < nst; ++s) { ss_mbar_init(&full_bar[s], 1); ss_mbar_init(&empty_bar[s], G::COLS4 / 32); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    const size_t img_floats = (size_t)P.rowlen * P.rows;
    uint32_t stage = 0, phase = 0;

    if (tid >= G::COLS4) {
        if (tid != G::COLS4) return;
        // ── producer lane ──
        bool first_lap = true;
        for (uint32_t u = blockIdx.x; u < P.nunits; u += gridDim.x) {
            const uint32_t strip = u % P.strips, rest = u / P.strips;
            const uint32_t chunk = rest % P.chunks, img = rest / P.chunks;
            const int e0 = (int)(strip * G::EW);
            const int g0 = max(e0 - HL, 0), g1 = min(e0 + G::EW + HR, (int)P.rowlen);  // floats, multiples of 4
            const uint32_t bytes = (uint32_t)(g1 - g0) * 4u;
            const uint32_t slot_off = (uint32_t)(g0 - (e0 - HL));                        // floats into the slot
            const int y_first = (int)(chunk * P.rows_per_chunk), y_end = min(y_first + (int)P.rows_per_chunk, (int)P.rows);
            const float* base = src + (size_t)img * img_floats + g0;
            for (int iy = y_first - HY; iy < y_end + (KY - 1 - HY); ++iy) {
                if (!first_lap) ss_mbar_wait(&empty_bar[stage], phase ^ 1u);
                const bool valid = iy >= 0 && iy < (int)P.rows;
                row_valid[stage] = valid ? 1 : 0;
                if (valid) {
                    ss_mbar_expect_tx(&full_bar[stage], bytes);
                    ss_tma_load_1d(ss_smem + (size_t)stage * P.slot_floats + slot_off, base + (size_t)iy * P.rowlen, bytes, &full_bar[stage]);
                } else {
                    ss_mbar_arrive(&full_bar[stage]);
                }
                if (++stage == nst) { stage = 0; phase ^= 1u; first_lap = false; }
            }
        }
        return;
    }

    // ── consumers: NV float4 columns each ──
    PairConst pc;
    pc.nz = ss_pack(R.neg_zero, R.neg_zero); pc.one = ss_pack(R.one, R.one); pc.zero = ss_pack(0.0f, 0.0f);
    ss_u64 kyp[SOBEL ? 1 : KY];
    if constexpr (!SOBEL) {
#pragma unroll
        for (int t = 0; t < KY; ++t) kyp[t] = ss_pack(taps.ky[t], taps.ky[t]);
    }
    const bool lane0 = (tid & 31u) == 0;

    // one unit (strip x row chunk) for this thread; EDGE = the strip touches the left or right image border (float4s
    // outside the row are zeroed in registers), interior strips carry no bounds logic at all
    auto consume = [&](auto edge_tag, int e0, int y_first, int y_end, float* __restrict__ out) {
        constexpr bool EDGE = decltype(edge_tag)::value;
        const int e = e0 + 4 * (int)tid;                 // first global float of this thread's column 0
        bool act[NV];
#pragma unroll
        for (int v = 0; v < NV; ++v) act[v] = !EDGE || (e + v * (G::COLS4 * 4) < (int)P.rowlen);
        ss_u64 winA[KY][NV][2], winB[SOBEL ? KY : 1][NV][2];
#pragma unroll
        for (int t = 0; t < KY; ++t)
#pragma unroll
            for (int v = 0; v < NV; ++v) { winA[t][v][0] = winA[t][v][1] = pc.zero; if (SOBEL) winB[t][v][0] = winB[t][v][1] = pc.zero; }
        int iy = y_first - HY;
        const int iy_end = y_end + (KY - 1 - HY);
        while (iy < iy_end) {
#pragma unroll
            for (int s = 0; s < KY; ++s) {   // unrolled: window slot indices are compile-time
                if (iy >= iy_end) break;
                ss_mbar_wait(&full_bar[stage], phase);
                const bool valid = row_valid[stage] != 0;
                const float4* sp = reinterpret_cast<const float4*>(ss_smem + (size_t)stage * P.slot_floats) + tid;
#pragma unroll
                for (int v = 0; v < NV; ++v) {
                    float hA[4] = {0.0f, 0.0f, 0.0f, 0.0f}, hB[4] = {0.0f, 0.0f, 0.0f, 0.0f};
                    if (valid && act[v]) {
                        float in[NF4 * 4];
#pragma unroll
                        for (int q = 0; q < NF4; ++q) {
                            float4 x = sp[v * G::COLS4 + q];
                            if (EDGE) {
                                const int gi = e + v * (G::COLS4 * 4) - HL + 4 * q;   // global float index of this float4
                                if (gi < 0 || gi >= (int)P.rowlen) x = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
                            }
                            in[4 * q] = x.x; in[4 * q + 1] = x.y; in[4 * q + 2] = x.z; in[4 * q + 3] = x.w;
                        }
#pragma unroll
                        for (int j = 0; j < 4; ++j) {
                            if constexpr (SOBEL) {
                                auto get = [&](int t) { return in[OFF + j + t * C]; };
                                hA[j] = SobelAcc<KX, true, 0>::run(0.0f, get);    // derivative taps along x  (gx)
                                hB[j] = SobelAcc<KX, false, 0>::run(0.0f, get);   // smoothing taps along x   (gy)
                            } else {
                                float a = fmaf(in[OFF + j], taps.kx[0], 0.0f);   // == 0 + in*k
#pragma unroll
                                for (int t = 1; t < KX; ++t) a += in[OFF + j + t * C] * taps.kx[t];
                                hA[j] = a;
                            }
                        }
                    }
                    winA[s][v][0] = ss_pack(hA[0], hA[1]); winA[s][v][1] = ss_pack(hA[2], hA[3]);
                    if (SOBEL) { winB[s][v][0] = ss_pack(hB[0], hB[1]); winB[s][v][1] = ss_pack(hB[2], hB[3]); }
                }
                __syncwarp();
                if (lane0) ss_mbar_arrive(&empty_bar[stage]);
                if (++stage == nst) { stage = 0; phase ^= 1u; }
                // the row that just became complete: r = iy - (KY-1-HY); its window is slots s+1 … s+KY (mod KY), oldest first
                if (iy - (KY - 1 - HY) >= y_first) {
#pragma unroll
                    for (int v = 0; v < NV; ++v) {
                        if (!act[v]) continue;
                        float o[4];
#pragma unroll
                        for (int h = 0; h < 2; ++h) {
                            if constexpr (SOBEL) {
                                auto getA = [&](int t) { return winA[(s + 1 + t) % KY][v][h]; };
                                auto getB = [&](int t) { return winB[(s + 1 + t) % KY][v][h]; };
                                const ss_u64 gx = SobelAccPair<KY, false, 0>::run(pc.zero, pc, getA);  // smoothing along y
                                const ss_u64 gy = SobelAccPair<KY, true, 0>::run(pc.zero, pc, getB);   // derivative along y
                                const ss_u64 m = pair_add(pair_mul(gx, gx, pc), pair_mul(gy, gy, pc), pc);   // gx*gx + gy*gy, unfused
                                float m0, m1;
                                ss_unpack(m, m0, m1);
                                pair_sqrt_rn(m0, m1, &o[2 * h], &o[2 * h + 1]);     // == sqrtf on both (pair_math.cuh)
                            } else {
                                ss_u64 acc = ss_fma2(winA[(s + 1) % KY][v][h], kyp[0], pc.zero);   // == 0 + w*k
#pragma unroll
                                for (int t = 1; t < KY; ++t) acc = pair_add(acc, pair_mul(winA[(s + 1 + t) % KY][v][h], kyp[t], pc), pc);
                                ss_unpack(acc, o[2 * h], o[2 * h + 1]);
                            }
                        }
                        stg_stream_f4(reinterpret_cast<float4*>(out + v * (G::COLS4 * 4)), make_float4(o[0], o[1], o[2], o[3]));
                    }
                    out += P.rowlen;
                }
                ++iy;
            }
        }
    };

    for (uint32_t u = blockIdx.x; u < P.nunits; u += gridDim.x) {
        const uint32_t strip = u % P.strips, rest = u / P.strips;
        const uint32_t chunk = rest % P.chunks, img = rest / P.chunks;
        const int e0 = (int)(strip * G::EW);
        const bool edge_unit = (e0 - HL < 0) || (e0 + G::EW + HR > (int)P.rowlen);
        const int y_first = (int)(chunk * P.rows_per_chunk), y_end = min(y_first + (int)P.rows_per_chunk, (int)P.rows);
        float* out = dst + (size_t)img * img_floats + (size_t)y_first * P.rowlen + e0 + 4 * (int)tid;
        if (edge_unit) consume(std::true_type{}, e0, y_first, y_end, out);
        else consume(std::false_type{}, e0, y_first, y_end, out);
    }
}

template <int C, int KX, int KY, bool SOBEL, int NV>
static int launch_sep_stream2(cudaStream_t s, const float* src, float* dst, const SepTaps& taps, uint32_t cols, uint32_t rows,
                              uint32_t batch) {
    using G = SS2<NV>;
    constexpr int HX = KX / 2;
    constexpr int HL = ((HX * C + 3) / 4) * 4, HR = (((KX - 1 - HX) * C + 3) / 4) * 4;
    const int tune_stages = knob(KNOB_SS_STAGES), tune_ctas = knob(KNOB_SS_CTAS);   // developer sweeps only (kb200_debug_set_knob)
    SepStream2Params R;
    SepStreamParams& P = R.g;
    P.rowlen = cols * C; P.rows = rows; P.batch = batch;
    P.strips = (P.rowlen + G::EW - 1) / G::EW;
    P.slot_floats = G::EW + HL + HR;
    // H100 sweep (16 x 4K f32, CTAs 3..10 x stages 2..6): blur is best at 6 CTAs x 4 stages, sobel at 4 x 4 (its
    // neighbours within 1 %; the 7 x 3 of the previous target is slower here).  Knobs ss.ctas / ss.stages re-sweep them.
    const uint32_t stages = (tune_stages >= 2 && tune_stages <= G::MAX_STAGES) ? (uint32_t)tune_stages : 4u;
    const int per_sm = tune_ctas > 0 ? tune_ctas : (SOBEL ? 4 : 6);
    const size_t smem = (size_t)P.slot_floats * 4 * stages;
    auto kern = sep_filter_stream2_kernel<C, KX, KY, SOBEL, NV>;
    if (smem > 40 * 1024) {
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return fail(KB200_ERR_CUDA, "cudaFuncSetAttribute(smem=%zu) failed: %s", smem, cudaGetErrorString(e));
    }
    // persistent CTAs must all be co-resident: never ask for more per SM than the occupancy calculator grants
    int resident = 0;
    {
        cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&resident, kern, G::THREADS, smem);
        if (e != cudaSuccess || resident < 1) return fail(KB200_ERR_CUDA, "occupancy query failed: %s", cudaGetErrorString(e));
    }
    const size_t ctas = (size_t)device_info().sm_count * std::min(per_sm, resident);
    // chunk height: ~12 units per CTA keeps the persistent grid balanced (a search that traded balance against the
    // KY-1 halo rows per chunk measured slower: long chunks leave the ragged last strip's CTAs idle);
    // at least 32 rows so the halo re-reads stay near 10 %
    const int tune_rc = knob(KNOB_SS_RC);
    const size_t total = (size_t)P.strips * batch * rows;
    uint32_t rc = tune_rc > 0 ? (uint32_t)tune_rc : (uint32_t)std::max<size_t>(32, total / (ctas * 12));
    rc = std::min(rc, rows);
    P.rows_per_chunk = rc;
    P.chunks = (rows + rc - 1) / rc;
    const size_t nunits = (size_t)P.strips * P.chunks * batch;
    if (nunits > 0x7FFFFFFFull) return fail(KB200_ERR_DIMS_TOO_LARGE, "too many filter work units (%zu)", nunits);
    P.nunits = (uint32_t)nunits;
    R.stages = stages;
    R.neg_zero = -0.0f; R.one = 1.0f;
    const unsigned grid = (unsigned)std::min<size_t>(nunits, ctas);
    kern<<<grid, G::THREADS, smem, s>>>(src, dst, taps, R);
    return check_launch("sep_filter_stream2_kernel");
}

// returns true if a streaming instance exists for (C, kx, ky, sobel) and launched it (status in *st)
static bool try_sep_stream(cudaStream_t s, const float* src, float* dst, const SepTaps& taps, uint32_t cols, uint32_t rows,
                           uint32_t C, uint32_t batch, bool sobel, int* st) {
    if (((size_t)cols * C) % 4 != 0 || !aligned16(src) || !aligned16(dst) || (size_t)cols * C < 16) return false;
    const int kx = taps.kxn, ky = taps.kyn;
#define KB200_SS_CASE(CC, KK, SB)                                                             \
    if (C == CC && kx == KK && ky == KK && sobel == SB) {                                     \
        *st = launch_sep_stream2<CC, KK, KK, SB, 1>(s, src, dst, taps, cols, rows, batch);    \
        return true;                                                                          \
    }
    KB200_SS_CASE(3, 5, false) KB200_SS_CASE(3, 3, false) KB200_SS_CASE(3, 7, false)
    KB200_SS_CASE(1, 5, false) KB200_SS_CASE(1, 3, false) KB200_SS_CASE(1, 7, false)
    KB200_SS_CASE(4, 5, false) KB200_SS_CASE(4, 3, false)
    KB200_SS_CASE(3, 3, true) KB200_SS_CASE(3, 5, true) KB200_SS_CASE(1, 3, true) KB200_SS_CASE(1, 5, true)
#undef KB200_SS_CASE
    return false;
}

// cuda/filter.rs:515-530
__global__ void gradient_magnitude_kernel(const float* __restrict__ gx, const float* __restrict__ gy,
                                          float* __restrict__ dst, size_t n) {
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const float a = __ldg(gx + i), b = __ldg(gy + i);
        dst[i] = sqrtf(a * a + b * b);
    }
}

template <int KX, int KY, bool SOBEL>
static int launch_sep_instance(cudaStream_t s, const float* src, float* dst, const SepTaps& taps, const SepGeom& g,
                               uint32_t batch, size_t smem_bytes) {
    auto kern = sep_filter_fused_kernel<KX, KY, SOBEL>;
    if (smem_bytes > 40 * 1024) {
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes);
        if (e != cudaSuccess) return fail(KB200_ERR_CUDA, "cudaFuncSetAttribute(smem=%zu) failed: %s", smem_bytes, cudaGetErrorString(e));
    }
    const size_t ntiles = (size_t)g.tiles_x * g.tiles_y * batch;
    if (ntiles > 0x7FFFFFFFull) return fail(KB200_ERR_DIMS_TOO_LARGE, "too many tiles (%zu)", ntiles);
    kern<<<(unsigned)ntiles, 256, smem_bytes, s>>>(src, dst, taps, g);
    return check_launch("sep_filter_fused_kernel");
}

static int launch_sep(cudaStream_t s, const float* src, size_t src_len, float* dst, size_t dst_len, const float* kx,
                      uint32_t kxn, const float* ky, uint32_t kyn, uint32_t cols, uint32_t rows, uint32_t C,
                      uint32_t batch, bool sobel) {
    KB200_TRY(check_ptr("src", src)); KB200_TRY(check_ptr("dst", dst));
    KB200_TRY(check_geometry(cols, rows, cols, rows, batch));
    if (C == 0 || kxn == 0 || kyn == 0) return fail(KB200_ERR_INVALID_KERNEL, "channels and tap counts must be at least 1");  // cuda/filter.rs:306-310
    if (C > 4) return fail(KB200_ERR_UNSUPPORTED, "separable filter supports 1..4 channels, got %u", C);
    if (kxn > (uint32_t)KB200_MAX_TAPS || kyn > (uint32_t)KB200_MAX_TAPS)
        return fail(KB200_ERR_UNSUPPORTED, "separable filter supports up to %d taps per axis, got (%u, %u)", KB200_MAX_TAPS, kxn, kyn);
    const size_t n = (size_t)cols * rows * C * batch;
    KB200_TRY(check_slice("src", src_len, n)); KB200_TRY(check_slice("dst", dst_len, n));
    if (src == dst) return fail(KB200_ERR_INVALID_ARGUMENT, "src and dst must not alias (tiles read a halo)");
    SepTaps taps{};
    for (uint32_t i = 0; i < kxn; ++i) taps.kx[i] = kx[i];
    for (uint32_t i = 0; i < kyn; ++i) taps.ky[i] = ky[i];
    taps.kxn = (int)kxn; taps.kyn = (int)kyn;
    {
        int st = KB200_OK;
        if (try_sep_stream(s, src, dst, taps, cols, rows, C, batch, sobel, &st)) return st;
    }
    SepGeom g;
    g.cols = cols; g.rows = rows; g.C = C;
    g.tw = 64; g.th = 32;
    if (cols <= 32) g.tw = 32;
    if (rows <= 16) g.th = 16;
    auto smem_for = [&](uint32_t tw, uint32_t th) {
        const size_t in_w = (size_t)(tw + kxn - 1) * C, in_h = th + kyn - 1, mid_w = (size_t)tw * C;
        return (in_w * in_h + mid_w * in_h * (sobel ? 2 : 1)) * sizeof(float);
    };
    size_t smem = smem_for(g.tw, g.th);
    const size_t cap = std::min<size_t>((size_t)device_info().max_smem_optin, 100 * 1024);
    while (smem > cap && (g.tw > 16 || g.th > 8)) {
        if (g.th > 8 && g.th >= g.tw / 2) g.th /= 2; else g.tw /= 2;
        smem = smem_for(g.tw, g.th);
    }
    if (smem > cap) return fail(KB200_ERR_UNSUPPORTED, "filter tile does not fit shared memory (%zu B)", smem);
    g.tiles_x = (cols + g.tw - 1) / g.tw;
    g.tiles_y = (rows + g.th - 1) / g.th;
    if (sobel) {
        if (kxn == 3) return launch_sep_instance<3, 3, true>(s, src, dst, taps, g, batch, smem);
        return launch_sep_instance<5, 5, true>(s, src, dst, taps, g, batch, smem);
    }
    if (kxn == 3 && kyn == 3) return launch_sep_instance<3, 3, false>(s, src, dst, taps, g, batch, smem);
    if (kxn == 5 && kyn == 5) return launch_sep_instance<5, 5, false>(s, src, dst, taps, g, batch, smem);
    if (kxn == 7 && kyn == 7) return launch_sep_instance<7, 7, false>(s, src, dst, taps, g, batch, smem);
    return launch_sep_instance<0, 0, false>(s, src, dst, taps, g, batch, smem);
}

}  // namespace kb200

using namespace kb200;

extern "C" {

KB200_API int kb200_separable_filter_f32(kb200_stream_t stream, const float* src, size_t src_len, float* dst,
                                         size_t dst_len, float* /*scratch*/, const float* kx, uint32_t kx_len,
                                         const float* ky, uint32_t ky_len, uint32_t cols, uint32_t rows,
                                         uint32_t channels, uint32_t batch) {
    KB200_TRY(check_ptr("kx", kx)); KB200_TRY(check_ptr("ky", ky));
    return launch_sep(as_stream(stream), src, src_len, dst, dst_len, kx, kx_len, ky, ky_len, cols, rows, channels, batch, false);
}

KB200_API int kb200_gaussian_blur_f32(kb200_stream_t stream, const float* src, size_t src_len, float* dst,
                                      size_t dst_len, uint32_t cols, uint32_t rows, uint32_t channels,
                                      uint32_t batch, uint32_t ksize_x, uint32_t ksize_y, float sigma_x,
                                      float sigma_y) {
    uint32_t kxn, kyn;
    float sx, sy;
    KB200_TRY(kb200_gaussian_resolve(ksize_x, ksize_y, sigma_x, sigma_y, &kxn, &kyn, &sx, &sy));
    if (kxn > (uint32_t)KB200_MAX_TAPS || kyn > (uint32_t)KB200_MAX_TAPS)
        return fail(KB200_ERR_UNSUPPORTED, "gaussian_blur supports up to %d taps per axis, got (%u, %u)", KB200_MAX_TAPS, kxn, kyn);
    float kx[32], ky[32];
    kb200_gaussian_kernel_1d(kxn, sx, kx);
    kb200_gaussian_kernel_1d(kyn, sy, ky);
    return launch_sep(as_stream(stream), src, src_len, dst, dst_len, kx, kxn, ky, kyn, cols, rows, channels, batch, false);
}

KB200_API int kb200_sobel_f32(kb200_stream_t stream, const float* src, size_t src_len, float* dst, size_t dst_len,
                              uint32_t cols, uint32_t rows, uint32_t channels, uint32_t batch, uint32_t ksize) {
    // filter/kernels.rs:55-72
    static const float d3[3] = {-1.0f, 0.0f, 1.0f}, s3[3] = {1.0f, 2.0f, 1.0f};
    static const float d5[5] = {-1.0f, -2.0f, 0.0f, 2.0f, 1.0f}, s5[5] = {1.0f, 4.0f, 6.0f, 4.0f, 1.0f};
    if (ksize != 3 && ksize != 5) return fail(KB200_ERR_INVALID_KERNEL, "invalid sobel kernel length %u (expected 3 or 5)", ksize);
    return launch_sep(as_stream(stream), src, src_len, dst, dst_len, ksize == 3 ? d3 : d5, ksize, ksize == 3 ? s3 : s5,
                      ksize, cols, rows, channels, batch, true);
}

KB200_API int kb200_gradient_magnitude_f32(kb200_stream_t stream, const float* gx, const float* gy, float* dst,
                                           size_t n) {
    KB200_TRY(check_ptr("gx", gx)); KB200_TRY(check_ptr("gy", gy)); KB200_TRY(check_ptr("dst", dst));
    if (n == 0) return KB200_OK;
    const unsigned grid = (unsigned)std::min<size_t>((n + 255) / 256, (size_t)device_info().sm_count * 16);
    gradient_magnitude_kernel<<<grid, 256, 0, as_stream(stream)>>>(gx, gy, dst, n);
    return check_launch("gradient_magnitude_kernel");
}

}  // extern "C"
