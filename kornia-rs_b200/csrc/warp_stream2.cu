// warp_stream2.cu — the bilinear fast consumer of the row-streaming warp design (config 5's kernel).
//
// Same producer, ring, schedule and queue discipline as warp_stream.cu (shared through warp_stream.cuh); what differs is
// the consumer loop, written for issue slots — SASS of the gather kernels showed ~70 INTEGER instructions per pixel
// (64-bit tap addresses, per-tap selects) against ~35 floating-point ones, and the generic streaming consumer is no
// leaner.  Here:
//   * a thread owns ONE destination column and processes TWO destination rows per step (the schedule is computed per
//     row pair, ws_pair_need), so mbarrier traffic, the named barrier and the row copy-out are paid once per two pixels;
//   * the two pixels are computed as a PAIR (fma2_rn, kb200_common.cuh): every `a*b` is fma2(a, b, -0) and every `a+b`
//     is fma2(a, 1, b) with -0 / 1 opaque kernel arguments — the reference's unfused, twice-rounded arithmetic;
//   * an interior pixel whose 2x2 footprint is resident takes its 12 taps as `LDS.32` at immediate offsets from TWO
//     32-bit shared-memory addresses (row y0 and row y0+1 of the ring) — no 64-bit address arithmetic, no per-tap select;
//   * everything else (image border pixels where a +1 neighbour is missing, a tap outside the resident band or span)
//     goes through `ws2_slow_pixel`, a non-inlined copy of the generic path (shared arithmetic: warp_common.cuh), so the
//     hot loop stays small.  Out-of-image pixels write 0.
#include <algorithm>
#include <cmath>

#include "warp_stream.cuh"

namespace kb200 {

typedef unsigned long long ws_u64;
__device__ __forceinline__ ws_u64 ws_pack(float a, float b) { ws_u64 r; asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(a), "f"(b)); return r; }
__device__ __forceinline__ void ws_unpack(ws_u64 v, float& a, float& b) { asm("mov.b64 {%0, %1}, %2;" : "=f"(a), "=f"(b) : "l"(v)); }
__device__ __forceinline__ ws_u64 ws_fma2(ws_u64 a, ws_u64 b, ws_u64 c) { return fma2_rn(a, b, c); }
struct WsConst { ws_u64 nz, one; };
__device__ __forceinline__ ws_u64 ws_mul(ws_u64 a, ws_u64 b, const WsConst& c) { return ws_fma2(a, b, c.nz); }
__device__ __forceinline__ ws_u64 ws_add(ws_u64 a, ws_u64 b, const WsConst& c) { return ws_fma2(a, c.one, b); }
__device__ __forceinline__ ws_u64 ws_bcast(float a) { return ws_pack(a, a); }
__device__ __forceinline__ float ws_lds(uint32_t addr) { float v; asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(addr)); return v; }

struct WarpStream2Args {
    WarpStreamParams p;
    float neg_zero, one;   // -0.0f and 1.0f, opaque to the optimiser on purpose
};

// Generic (checked) evaluation of one destination pixel: any edge rule, resident or not.  Rare path; never inlined.
struct Ws2Px { float v0, v1, v2; };

template <bool PERSPECTIVE>
__device__ __noinline__ Ws2Px ws2_slow_pixel(const WarpStreamParams& P, const float* __restrict__ gsrc, const float* ring, uint32_t gx, uint32_t dy,
                                             int rel_g, int ld_g, int c0, int span, uint32_t qoff) {
    Ws2Px o;
    o.v0 = 0.0f; o.v1 = 0.0f; o.v2 = 0.0f;
    float sx, sy;
    if (!warp_coord<PERSPECTIVE>(P.m, gx, dy, P.sw, P.sh, &sx, &sy)) return o;
    WarpTaps t;
    warp_taps<PERSPECTIVE, true>(sx, sy, P.sw, P.sh, &t);
    const int fa = (int)t.x0 * 3 - c0, fb = (int)t.x1 * 3 - c0;
    const bool in_ring = ld_g >= rel_g && (int)t.y0 >= rel_g && (int)t.y1 <= ld_g && (int)t.y1 >= rel_g && (int)t.y0 <= ld_g &&
                         fa >= 0 && fb >= 0 && fa + 3 <= span && fb + 3 <= span;
    if (in_ring) {
        const uint32_t smask = P.nslot - 1u;
        const float* ra = ring + (size_t)((qoff + t.y0) & smask) * P.slot_floats;
        const float* rb = ring + (size_t)((qoff + t.y1) & smask) * P.slot_floats;
        warp_blend<true>(t, ra + fa, ra + fb, rb + fa, rb + fb, &o.v0, &o.v1, &o.v2);
    } else {
        const float* ra = gsrc + (size_t)t.y0 * P.row_floats;
        const float* rb = gsrc + (size_t)t.y1 * P.row_floats;
        warp_blend_ldg<true>(t, ra + t.x0 * 3u, ra + t.x1 * 3u, rb + t.x0 * 3u, rb + t.x1 * 3u, &o.v0, &o.v1, &o.v2);
    }
    return o;
}

template <bool PERSPECTIVE>
__global__ void __launch_bounds__(WS_THREADS) warp_stream2_kernel(const float* __restrict__ src, float* __restrict__ dst,
                                                                  const __grid_constant__ WarpStream2Args A) {
    extern __shared__ __align__(128) float ws_smem[];
    __shared__ __align__(8) uint64_t full_bar[WS_MAX_SLOTS];
    __shared__ __align__(8) uint64_t empty_bar[WS_MAX_SLOTS];
    const WarpStreamParams& P = A.p;
    constexpr uint32_t TW = WS_CT;                 // one column per thread
    constexpr uint32_t ROW_FLOATS = TW * 3u;       // one destination row of the tile
    constexpr uint32_t OUT_FLOATS = ROW_FLOATS * 2u;   // a step writes two rows
    const uint32_t tid = threadIdx.x, lane = tid & 31u;
    const int nslot = (int)P.nslot;
    const uint32_t smask = P.nslot - 1u;
    float* ring = ws_smem + 2u * OUT_FLOATS;       // [2 x (2 out rows)][ring]
    const size_t src_img = (size_t)P.row_floats * P.sh, dst_img = (size_t)P.dw * P.dh * 3u;

    if (tid == 0) {
        for (uint32_t s = 0; s < P.nslot; ++s) { tma::mbar_init(&full_bar[s], 1); tma::mbar_init(&empty_bar[s], WS_CT / 32); }
        tma::mbar_fence_init();
    }
    __syncthreads();

    if (tid >= WS_CT) {
        ws_producer<PERSPECTIVE, true, TW>(src, P, ring, full_bar, empty_bar);
        return;
    }

    // ── consumer warps ──
    WsConst pc;
    pc.nz = ws_bcast(A.neg_zero); pc.one = ws_bcast(A.one);
    const float* m = P.m;
    const float fsw = (float)P.sw, fsh = (float)P.sh;
    const uint32_t ring_u32 = tma::smem_u32(ring);
    const uint32_t slot_bytes = P.slot_floats * 4u;
    WSWalk w;
    w.init(blockIdx.x, P);
    uint32_t qbase = 0, obuf = 0;
    for (uint32_t u = blockIdx.x; u < P.nunits; u += gridDim.x, w.advance(P)) {
        const uint32_t dx0 = w.tx * TW, dx1 = min(dx0 + TW, P.dw) - 1u;
        const uint32_t y_first = w.cy * P.rows_per_chunk, y_end = min(y_first + P.rows_per_chunk, P.dh);
        int c0, c1;
        ws_span<PERSPECTIVE>(P, dx0, dx1, y_first, y_end - 1u, &c0, &c1);
        const int span = c1 - c0;
        const bool staged_unit = span > 0;
        const bool fast_unit = span >= 6;                       // room for one 2-pixel footprint
        const uint32_t colmax = fast_unit ? (uint32_t)(span - 6) : 0u;
        const float* gsrc = src + (size_t)w.img * src_img;
        float* grow = dst + (size_t)w.img * dst_img + ((size_t)y_first * P.dw + dx0) * 3u;
        const uint32_t valid_floats = (dx1 - dx0 + 1u) * 3u;
        const uint32_t gx = dx0 + tid;
        const bool col_on = gx < P.dw;
        const float x = (float)gx;
        // x-terms of the inverse map, shared by every row of the unit
        const ws_u64 ax = ws_bcast(m[0] * x), bx = ws_bcast(m[3] * x), cx = ws_bcast(PERSPECTIVE ? m[6] * x : 0.0f);
        const bool degx = fabsf(m[0]) < 1e-6f, degy = fabsf(m[3]) < 1e-6f;
        int r0 = -1, rel_c = 0, ld_c = -1, seen = -1;
        uint32_t qoff = 0;     // slot of source row r = (qoff + r) & smask
        for (uint32_t yb = y_first; yb < y_end; yb += 32u) {
            int lo, hi;
            ws_row_need<PERSPECTIVE>(P, dx0, dx1, yb + lane, yb + lane < y_end, &lo, &hi);
            ws_pair_need(&lo, &hi);
            bool have = r0 >= 0;
            if (!have) {
                int first = (lo <= hi) ? lo : 0x7FFFFFFF;
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) first = min(first, __shfl_xor_sync(0xFFFFFFFFu, first, o));
                if (first != 0x7FFFFFFF) { r0 = first; rel_c = first; ld_c = first - 1; seen = first - 1; have = true; qoff = qbase - (uint32_t)first; }
            }
            int rel = rel_c, ld = ld_c;
            if (have) ws_schedule(lo, hi, rel_c, ld_c, nslot, &rel, &ld);
            const uint32_t nrows = min(32u, y_end - yb);
            const bool ring_on = have && staged_unit;
            for (uint32_t i = 0; i < nrows; i += 2u) {
                const uint32_t yA = yb + i, yB = yA + 1u;
                const bool b_row = yB < y_end;
                const int rel_g = __shfl_sync(0xFFFFFFFFu, rel, (int)i), ld_g = __shfl_sync(0xFFFFFFFFu, ld, (int)i);   // identical on both lanes of the pair
                if (ring_on && (ld_g > seen || rel_g > rel_c)) {
                    // bounded-queue discipline (see warp_stream.cu): acquire in order, release in order, release before the
                    // wait that needs the slot back
                    for (int r = seen + 1; r <= ld_g; ++r) {
                        const int upto = min(rel_g, r - nslot + 1);
                        if (lane == 0) {
                            for (int k = rel_c; k < upto; ++k) tma::mbar_arrive(&empty_bar[(qoff + (uint32_t)k) & smask]);
                        }
                        rel_c = max(rel_c, upto);
                        const uint32_t q = qoff + (uint32_t)r;
                        tma::mbar_wait(&full_bar[q & smask], (q >> P.nslot_log2) & 1u);
                    }
                    seen = max(seen, ld_g);
                    if (lane == 0) {
                        for (int k = rel_c; k < rel_g; ++k) tma::mbar_arrive(&empty_bar[(qoff + (uint32_t)k) & smask]);
                    }
                    rel_c = max(rel_c, rel_g);
                }
                const uint32_t nres = (uint32_t)max(ld_g - rel_g, 0);   // rows y0 with y0 and y0+1 both resident: rel_g <= y0 < ld_g
                // ── two pixels (gx, yA) and (gx, yB) as a pair ──
                const ws_u64 y = ws_pack((float)yA, (float)yB);
                float sx[2], sy[2];
                bool ok[2];
                if (PERSPECTIVE) {
                    const ws_u64 w2 = ws_add(ws_add(cx, ws_mul(ws_bcast(m[7]), y, pc), pc), ws_bcast(m[8]), pc);
                    const ws_u64 nx = ws_add(ws_add(ax, ws_mul(ws_bcast(m[1]), y, pc), pc), ws_bcast(m[2]), pc);
                    const ws_u64 ny = ws_add(ws_add(bx, ws_mul(ws_bcast(m[4]), y, pc), pc), ws_bcast(m[5]), pc);
                    float wv[2], nxs[2], nys[2];
                    ws_unpack(w2, wv[0], wv[1]); ws_unpack(nx, nxs[0], nxs[1]); ws_unpack(ny, nys[0], nys[1]);
#pragma unroll
                    for (int k = 0; k < 2; ++k) {
                        sx[k] = __fdiv_rn(nxs[k], wv[k]);
                        sy[k] = __fdiv_rn(nys[k], wv[k]);
                        ok[k] = !(fabsf(wv[k]) < 1e-10f) && sx[k] >= 0.0f && sx[k] < fsw && sy[k] >= 0.0f && sy[k] < fsh;
                    }
                } else {
                    const ws_u64 sx0 = ws_add(ws_mul(ws_bcast(m[1]), y, pc), ws_bcast(m[2]), pc);
                    const ws_u64 sy0 = ws_add(ws_mul(ws_bcast(m[4]), y, pc), ws_bcast(m[5]), pc);
                    const ws_u64 sxp = ws_add(ax, sx0, pc), syp = ws_add(bx, sy0, pc);
                    float sx0s[2], sy0s[2];
                    ws_unpack(sx0, sx0s[0], sx0s[1]); ws_unpack(sy0, sy0s[0], sy0s[1]);
                    ws_unpack(sxp, sx[0], sx[1]); ws_unpack(syp, sy[0], sy[1]);
#pragma unroll
                    for (int k = 0; k < 2; ++k) {
                        const float tx = degx ? sx0s[k] : sx[k], ty = degy ? sy0s[k] : sy[k];
                        ok[k] = tx >= 0.0f && tx < fsw && ty >= 0.0f && ty < fsh;
                    }
                }
                ok[0] = ok[0] && col_on;
                ok[1] = ok[1] && col_on && b_row;
                // taps: fast = interior pixel (both +1 neighbours exist) with a resident 2x2 footprint
                uint32_t a0[2], a1[2];
                float fx[2], fy[2];
                bool fast[2];
#pragma unroll
                for (int k = 0; k < 2; ++k) {
                    float sxc = sx[k], syc = sy[k];
                    if (!PERSPECTIVE) {   // per-axis clamp (cuda/warp_affine.rs:120-123); a valid perspective coordinate is already in range
                        sxc = fmaxf(fminf(sxc, (float)(P.sw - 1u)), 0.0f);
                        syc = fmaxf(fminf(syc, (float)(P.sh - 1u)), 0.0f);
                    }
                    const uint32_t x0 = (uint32_t)sxc, y0 = (uint32_t)syc;
                    fx[k] = sxc - (float)x0; fy[k] = syc - (float)y0;
                    const int fa = (int)(x0 * 3u) - c0;
                    const bool interior = (x0 + 1u) < P.sw && (y0 + 1u) < P.sh;
                    const bool resident = ring_on && fast_unit && (uint32_t)((int)y0 - rel_g) < nres && (uint32_t)fa <= colmax;
                    fast[k] = ok[k] && interior && resident;
                    const uint32_t s0 = fast[k] ? ((qoff + y0) & smask) : 0u, s1 = fast[k] ? ((qoff + y0 + 1u) & smask) : 0u;
                    const uint32_t off = fast[k] ? (uint32_t)fa * 4u : 0u;
                    a0[k] = ring_u32 + s0 * slot_bytes + off;
                    a1[k] = ring_u32 + s1 * slot_bytes + off;
                }
                const ws_u64 fxp = ws_pack(fx[0], fx[1]), fyp = ws_pack(fy[0], fy[1]);
                const ws_u64 neg1 = ws_bcast(-1.0f), one1 = ws_bcast(1.0f);
                const ws_u64 fxx = ws_fma2(fxp, neg1, one1), fyy = ws_fma2(fyp, neg1, one1);   // 1 - f: one rounding either way
                const ws_u64 w00 = ws_mul(fxx, fyy, pc), w10 = ws_mul(fxp, fyy, pc), w01 = ws_mul(fxx, fyp, pc), w11 = ws_mul(fxp, fyp, pc);
                float outA[3], outB[3];
                // One vote per step: if every lane's two pixels are either out of the image or on the fast path, the step is
                // straight-line code; a single slow pixel anywhere in the warp sends the whole step through the checked path.
                const bool lane_fast = (fast[0] || !ok[0]) && (fast[1] || !ok[1]);
                if (__all_sync(0xFFFFFFFFu, lane_fast)) {
#pragma unroll
                    for (int c = 0; c < 3; ++c) {
                        // (x0,y0) (x1,y0) (x0,y1) (x1,y1): immediate offsets 0 / 12 bytes from the two row addresses
                        const ws_u64 v00 = ws_pack(ws_lds(a0[0] + 4u * c), ws_lds(a0[1] + 4u * c));
                        const ws_u64 v10 = ws_pack(ws_lds(a0[0] + 12u + 4u * c), ws_lds(a0[1] + 12u + 4u * c));
                        const ws_u64 v01 = ws_pack(ws_lds(a1[0] + 4u * c), ws_lds(a1[1] + 4u * c));
                        const ws_u64 v11 = ws_pack(ws_lds(a1[0] + 12u + 4u * c), ws_lds(a1[1] + 12u + 4u * c));
                        ws_u64 acc = ws_mul(w00, v00, pc);
                        acc = ws_add(acc, ws_mul(w10, v10, pc), pc);
                        acc = ws_add(acc, ws_mul(w01, v01, pc), pc);
                        acc = ws_add(acc, ws_mul(w11, v11, pc), pc);
                        ws_unpack(acc, outA[c], outB[c]);
                    }
#pragma unroll
                    for (int c = 0; c < 3; ++c) { outA[c] = ok[0] ? outA[c] : 0.0f; outB[c] = ok[1] ? outB[c] : 0.0f; }
                } else {
                    Ws2Px pa, pb;
                    pa.v0 = pa.v1 = pa.v2 = 0.0f; pb = pa;
                    if (ok[0]) pa = ws2_slow_pixel<PERSPECTIVE>(P, gsrc, ring, gx, yA, ring_on ? rel_g : 0, ring_on ? ld_g : -1, c0, span, qoff);
                    if (ok[1]) pb = ws2_slow_pixel<PERSPECTIVE>(P, gsrc, ring, gx, yB, ring_on ? rel_g : 0, ring_on ? ld_g : -1, c0, span, qoff);
                    outA[0] = pa.v0; outA[1] = pa.v1; outA[2] = pa.v2;
                    outB[0] = pb.v0; outB[1] = pb.v1; outB[2] = pb.v2;
                }
                if (P.vec_store) {
                    float* orow = ws_smem + obuf * OUT_FLOATS + tid * 3u;
                    orow[0] = outA[0]; orow[1] = outA[1]; orow[2] = outA[2];
                    orow[ROW_FLOATS] = outB[0]; orow[ROW_FLOATS + 1u] = outB[1]; orow[ROW_FLOATS + 2u] = outB[2];
                    tma::named_barrier(1, WS_CT);
                    // two rows of ROW_FLOATS / 4 = 96 float4 each: threads 0..95 copy row A, threads 32..127 copy row B
                    const float4* o4 = reinterpret_cast<const float4*>(ws_smem + obuf * OUT_FLOATS);
                    if (tid < ROW_FLOATS / 4u && tid * 4u < valid_floats) stg_stream_f4(reinterpret_cast<float4*>(grow) + tid, o4[tid]);
                    const uint32_t tb = tid - (WS_CT - ROW_FLOATS / 4u);
                    if (b_row && tid >= WS_CT - ROW_FLOATS / 4u && tb * 4u < valid_floats)
                        stg_stream_f4(reinterpret_cast<float4*>(grow + (size_t)P.dw * 3u) + tb, o4[ROW_FLOATS / 4u + tb]);
                    obuf ^= 1u;
                } else if (col_on) {
                    float* q = grow + (size_t)tid * 3u;
                    q[0] = outA[0]; q[1] = outA[1]; q[2] = outA[2];
                    if (b_row) { q += (size_t)P.dw * 3u; q[0] = outB[0]; q[1] = outB[1]; q[2] = outB[2]; }
                }
                grow += (size_t)P.dw * 6u;
            }
            if (have) { rel_c = max(rel_c, __shfl_sync(0xFFFFFFFFu, rel, 31)); ld_c = max(ld_c, __shfl_sync(0xFFFFFFFFu, ld, 31)); }
        }
        if (r0 >= 0 && staged_unit) {
            for (int r = seen + 1; r <= ld_c; ++r) {
                const uint32_t q = qoff + (uint32_t)r;
                tma::mbar_wait(&full_bar[q & smask], (q >> P.nslot_log2) & 1u);
            }
            __syncwarp();
            if (lane == 0) {
                for (int k = rel_c; k <= ld_c; ++k) tma::mbar_arrive(&empty_bar[(qoff + (uint32_t)k) & smask]);
            }
            qbase += (uint32_t)(ld_c - r0 + 1);
        }
    }
}

// launched by launch_warp_stream (warp_stream.cu) for bilinear maps; same planning, one column per thread
template <bool PERSPECTIVE>
int ws2_launch(cudaStream_t s, const float* src, float* dst, WarpStreamParams& P, uint32_t batch, int per_sm_want, uint32_t rc_want, bool* handled) {
    auto kern = warp_stream2_kernel<PERSPECTIVE>;
    constexpr uint32_t TW = WS_CT;
    const size_t smem = (size_t)TW * 3u * 4u * 4u + (size_t)P.nslot * P.slot_floats * 4u;
    if (smem > 200 * 1024) return KB200_OK;
    if (smem > 40 * 1024 && cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) { cudaGetLastError(); return KB200_OK; }
    int resident = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&resident, kern, WS_THREADS, smem) != cudaSuccess || resident < 1) { cudaGetLastError(); return KB200_OK; }
    const int per_sm = std::min(per_sm_want, resident);
    P.tiles_x = (P.dw + TW - 1) / TW;
    const size_t ctas = (size_t)device_info().sm_count * per_sm;
    const size_t total_rows = (size_t)P.dh * batch * P.tiles_x;
    uint32_t rc = rc_want ? rc_want : (uint32_t)std::max<size_t>(96, total_rows / (ctas * 8));
    rc = std::min((rc + 1u) & ~1u, P.dh);     // even: row pairs never straddle a chunk
    P.rows_per_chunk = rc;
    P.chunks_y = (P.dh + rc - 1) / rc;
    const size_t nunits = (size_t)P.tiles_x * P.chunks_y * batch;
    if (nunits > 0x7FFFFFFFull) return KB200_OK;
    P.nunits = (uint32_t)nunits;
    const unsigned grid = (unsigned)std::min<size_t>(nunits, ctas);
    P.dtx = grid % P.tiles_x;
    const uint32_t g = grid / P.tiles_x;
    P.dcy = g % P.chunks_y;
    P.dimg = g / P.chunks_y;
    WarpStream2Args A;
    A.p = P; A.neg_zero = -0.0f; A.one = 1.0f;
    kern<<<grid, WS_THREADS, smem, s>>>(src, dst, A);
    KB200_TRY(check_launch("warp_stream2_kernel"));
    *handled = true;
    return KB200_OK;
}

template int ws2_launch<false>(cudaStream_t, const float*, float*, WarpStreamParams&, uint32_t, int, uint32_t, bool*);
template int ws2_launch<true>(cudaStream_t, const float*, float*, WarpStreamParams&, uint32_t, int, uint32_t, bool*);

}  // namespace kb200
