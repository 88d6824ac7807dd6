// warp_stream.cu — row-streaming warp_affine / warp_perspective (f32 HWC C=3) for gentle maps (config 5).
//
// Reference: cuda/warp_perspective.rs:51-167, cuda/warp_affine.rs:74-230 (one thread per destination pixel, 12 scattered
// `__ldg` taps).  ncu on our own gather kernels showed that design bound by memory LATENCY: a thread brings in 12 new bytes per pixel, so ~25 KB of unique bytes are in flight per SM.  Here
// the source is streamed instead of gathered:
//
//   * work unit = (image, tile of TW = 128*NPX destination columns, chunk of destination rows); persistent CTAs.
//   * the inverse map of a near-identity homography / small rotation sends a destination row segment to a thin BAND of
//     source rows that slides down by about one row per destination row.  A producer warp walks that band: every source
//     row span the tile needs is copied global -> shared exactly once by the TMA engine (`cp.async.bulk`, SASS UBLKCP)
//     into a ring of NSLOT row slots (slot = load sequence number mod NSLOT), completion counted on the slot's `full`
//     mbarrier; consumers release a slot (`empty` mbarrier) when the band has moved past its row.  Bytes in flight per SM
//     are set by the ring, not by the thread count, and every DRAM access is a whole-line bulk copy.
//   * the row SCHEDULE (which source rows must be resident before destination row dy, which may be dropped) is computed
//     32 destination rows at a time, one row per lane, from the two end pixels of the segment (a projective map is
//     monotone along a line), by the producer warp and by every consumer warp with the same instructions — so both sides
//     agree without communicating.  The schedule only has to be CONSISTENT: a tap that is not resident (rounding at the
//     band edge, a band taller than the ring, a span wider than a slot) is read from global memory instead, so the
//     staging can never change a result.
//   * 4 consumer warps; a thread owns NPX lane-contiguous destination columns for the whole unit (x-terms of the inverse
//     map in registers); taps are `LDS.32` from the ring; the destination row is assembled in shared memory and leaves as
//     lane-contiguous `STG.128`.
//
// Arithmetic: the expression trees of cuda/warp_perspective.rs:67-119 / cuda/warp_affine.rs:93-153 (unfused, IEEE
// division, validity rules, the two different edge rules) — `warp_coord` and the tap/weight code are shared with the
// gather kernels in warp.cu through warp_common.cuh, so all variants are the same arithmetic by construction.
#include <algorithm>
#include <cmath>

#include "warp_stream.cuh"

namespace kb200 {

template <bool PERSPECTIVE, bool BILINEAR, int NPX>
__global__ void __launch_bounds__(WS_THREADS) warp_stream_kernel(const float* __restrict__ src, float* __restrict__ dst,
                                                                 const __grid_constant__ WarpStreamParams P) {
    extern __shared__ __align__(128) float ws_smem[];
    __shared__ __align__(8) uint64_t full_bar[WS_MAX_SLOTS];
    __shared__ __align__(8) uint64_t empty_bar[WS_MAX_SLOTS];
    constexpr uint32_t TW = WS_CT * NPX;
    constexpr uint32_t OUT_FLOATS = TW * 3u;
    const uint32_t tid = threadIdx.x, lane = tid & 31u;
    const int nslot = (int)P.nslot;
    const uint32_t smask = P.nslot - 1u;
    float* ring = ws_smem + 2u * OUT_FLOATS;
    const size_t src_img = (size_t)P.row_floats * P.sh, dst_img = (size_t)P.dw * P.dh * 3u;

    if (tid == 0) {
        for (uint32_t s = 0; s < P.nslot; ++s) { tma::mbar_init(&full_bar[s], 1); tma::mbar_init(&empty_bar[s], WS_CT / 32); }
        tma::mbar_fence_init();
    }
    __syncthreads();

    WSWalk w;
    w.init(blockIdx.x, P);
    // Load sequence numbers: the q-th row this CTA loads lives in slot q & smask, phase (q / nslot) & 1.  Within a unit,
    // source row r has q = qbase + (r - r0) with r0 the unit's first resident row; qbase continues across units.
    uint32_t qbase = 0;

    if (tid >= WS_CT) {
        ws_producer<PERSPECTIVE, false, TW>(src, P, ring, full_bar, empty_bar);
        return;
    }

    // ── consumer warps ──
    uint32_t obuf = 0;
    for (uint32_t u = blockIdx.x; u < P.nunits; u += gridDim.x, w.advance(P)) {
        const uint32_t dx0 = w.tx * TW, dx1 = min(dx0 + TW, P.dw) - 1u;
        const uint32_t y_first = w.cy * P.rows_per_chunk, y_end = min(y_first + P.rows_per_chunk, P.dh);
        int c0, c1;
        ws_span<PERSPECTIVE>(P, dx0, dx1, y_first, y_end - 1u, &c0, &c1);
        const bool staged_unit = c1 > c0;
        const float* gsrc = src + (size_t)w.img * src_img;
        float* grow = dst + (size_t)w.img * dst_img + ((size_t)y_first * P.dw + dx0) * 3u;
        const uint32_t valid_px = dx1 - dx0 + 1u;
        uint32_t gxs[NPX];
#pragma unroll
        for (int j = 0; j < NPX; ++j) gxs[j] = dx0 + tid + (uint32_t)j * WS_CT;
        int r0 = -1, rel_c = 0, ld_c = -1;
        int seen = -1;        // rows <= seen have been waited for (this warp)
        for (uint32_t yb = y_first; yb < y_end; yb += 32u) {
            int lo, hi;
            ws_row_need<PERSPECTIVE>(P, dx0, dx1, yb + lane, yb + lane < y_end, &lo, &hi);
            bool have = r0 >= 0;
            if (!have) {
                int first = (lo <= hi) ? lo : 0x7FFFFFFF;
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) first = min(first, __shfl_xor_sync(0xFFFFFFFFu, first, o));
                if (first != 0x7FFFFFFF) { r0 = first; rel_c = first; ld_c = first - 1; seen = first - 1; have = true; }
            }
            int rel = rel_c, ld = ld_c;
            if (have) ws_schedule(lo, hi, rel_c, ld_c, nslot, &rel, &ld);
            const uint32_t nrows = min(32u, y_end - yb);
            for (uint32_t i = 0; i < nrows; ++i) {
                const uint32_t dy = yb + i;
                const int rel_i = __shfl_sync(0xFFFFFFFFu, rel, (int)i), ld_i = __shfl_sync(0xFFFFFFFFu, ld, (int)i);
                const bool ring_on = have && staged_unit;
                if (ring_on) {
                    // Bounded queue discipline: rows are acquired (wait `full`) in order and released (arrive `empty`) in
                    // order, a row only after it was acquired.  The producer can load row r once row r - nslot is
                    // released, so before waiting for r everything up to r - nslot (< rel_i by the schedule's cap) is
                    // handed back first — no circular wait, whatever the map does.
                    for (int r = seen + 1; r <= ld_i; ++r) {
                        const int upto = min(rel_i, r - nslot + 1);
                        if (lane == 0) {
                            for (int k = rel_c; k < upto; ++k) tma::mbar_arrive(&empty_bar[(qbase + (uint32_t)(k - r0)) & smask]);
                        }
                        rel_c = max(rel_c, upto);
                        const uint32_t q = qbase + (uint32_t)(r - r0);
                        tma::mbar_wait(&full_bar[q & smask], (q >> P.nslot_log2) & 1u);
                    }
                    seen = max(seen, ld_i);
                    if (lane == 0) {
                        for (int k = rel_c; k < rel_i; ++k) tma::mbar_arrive(&empty_bar[(qbase + (uint32_t)(k - r0)) & smask]);
                    }
                    rel_c = max(rel_c, rel_i);
                }
                float* orow = ws_smem + obuf * OUT_FLOATS;
#pragma unroll
                for (int j = 0; j < NPX; ++j) {
                    const uint32_t gx = gxs[j];
                    float v0 = 0.0f, v1 = 0.0f, v2 = 0.0f;
                    float sx, sy;
                    if (gx < P.dw && warp_coord<PERSPECTIVE>(P.m, gx, dy, P.sw, P.sh, &sx, &sy)) {
                        WarpTaps t;
                        warp_taps<PERSPECTIVE, BILINEAR>(sx, sy, P.sw, P.sh, &t);
                        // resident iff both rows are in [rel_i, ld_i] and both columns inside the staged span
                        const int fa = (int)t.x0 * 3 - c0, fb = (int)t.x1 * 3 - c0;
                        const bool in_ring = ring_on && (int)t.y0 >= rel_i && (int)t.y1 <= ld_i && (int)t.y0 <= ld_i && (int)t.y1 >= rel_i &&
                                             fa >= 0 && fb >= 0 && fa + 3 <= c1 - c0 && fb + 3 <= c1 - c0;
                        if (in_ring) {
                            const float* ra = ring + (size_t)((qbase + (uint32_t)((int)t.y0 - r0)) & smask) * P.slot_floats;
                            const float* rb = ring + (size_t)((qbase + (uint32_t)((int)t.y1 - r0)) & smask) * P.slot_floats;
                            warp_blend<BILINEAR>(t, ra + fa, ra + fb, rb + fa, rb + fb, &v0, &v1, &v2);
                        } else {
                            const float* ra = gsrc + (size_t)t.y0 * P.row_floats;
                            const float* rb = gsrc + (size_t)t.y1 * P.row_floats;
                            warp_blend_ldg<BILINEAR>(t, ra + t.x0 * 3u, ra + t.x1 * 3u, rb + t.x0 * 3u, rb + t.x1 * 3u, &v0, &v1, &v2);
                        }
                    }
                    if (P.vec_store) {
                        float* q = orow + (tid + (uint32_t)j * WS_CT) * 3u;
                        q[0] = v0; q[1] = v1; q[2] = v2;
                    } else if (gx < P.dw) {
                        float* q = grow + (size_t)(tid + (uint32_t)j * WS_CT) * 3u;
                        q[0] = v0; q[1] = v1; q[2] = v2;
                    }
                }
                if (P.vec_store) {
                    tma::named_barrier(1, WS_CT);
                    const float4* o4 = reinterpret_cast<const float4*>(orow);
                    float4* g4 = reinterpret_cast<float4*>(grow);
#pragma unroll
                    for (uint32_t k = 0; k < (OUT_FLOATS / 4u + WS_CT - 1u) / WS_CT; ++k) {
                        const uint32_t v = tid + k * WS_CT;
                        if (v * 4u < valid_px * 3u) stg_stream_f4(g4 + v, o4[v]);
                    }
                    obuf ^= 1u;
                }
                grow += (size_t)P.dw * 3u;
            }
            if (have) { rel_c = max(rel_c, __shfl_sync(0xFFFFFFFFu, rel, 31)); ld_c = max(ld_c, __shfl_sync(0xFFFFFFFFu, ld, 31)); }
        }
        if (r0 >= 0 && staged_unit) {
            // end of unit: the producer loaded rows r0 .. ld_c; wait for the ones this warp never needed to look at (their
            // `full` phase must complete before the slot is handed back), then release everything still held
            for (int r = seen + 1; r <= ld_c; ++r) {
                const uint32_t q = qbase + (uint32_t)(r - r0);
                tma::mbar_wait(&full_bar[q & smask], (q >> P.nslot_log2) & 1u);
            }
            __syncwarp();
            if (lane == 0) {
                for (int r = rel_c; r <= ld_c; ++r) tma::mbar_arrive(&empty_bar[(qbase + (uint32_t)(r - r0)) & smask]);
            }
            qbase += (uint32_t)(ld_c - r0 + 1);
        }
    }
}

template <bool PERSPECTIVE, bool BILINEAR, int NPX>
static int ws_launch(cudaStream_t s, const float* src, float* dst, WarpStreamParams& P, uint32_t batch, int per_sm_want, uint32_t rc_want, bool* handled) {
    auto kern = warp_stream_kernel<PERSPECTIVE, BILINEAR, NPX>;
    constexpr uint32_t TW = WS_CT * NPX;
    const size_t smem = (size_t)TW * 3u * 4u * 2u + (size_t)P.nslot * P.slot_floats * 4u;
    if (smem > 200 * 1024) return KB200_OK;
    if (smem > 40 * 1024 && cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) { cudaGetLastError(); return KB200_OK; }
    int resident = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&resident, kern, WS_THREADS, smem) != cudaSuccess || resident < 1) { cudaGetLastError(); return KB200_OK; }
    const int per_sm = std::min(per_sm_want, resident);
    P.tiles_x = (P.dw + TW - 1) / TW;
    const size_t ctas = (size_t)device_info().sm_count * per_sm;
    // chunk height: long enough that re-reading the band at a chunk seam (~band height rows) stays a few percent,
    // short enough for ~8 units per CTA
    const size_t total_rows = (size_t)P.dh * batch * P.tiles_x;
    uint32_t rc = rc_want ? rc_want : (uint32_t)std::max<size_t>(96, total_rows / (ctas * 8));
    rc = std::min(rc, P.dh);
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
    kern<<<grid, WS_THREADS, smem, s>>>(src, dst, P);
    KB200_TRY(check_launch("warp_stream_kernel"));
    *handled = true;
    return KB200_OK;
}

template <bool PERSPECTIVE>
int ws2_launch(cudaStream_t s, const float* src, float* dst, WarpStreamParams& P, uint32_t batch, int per_sm_want, uint32_t rc_want, bool* handled);   // warp_stream2.cu

// Host-side applicability test + launch.  `minv`: inverse matrix (9 floats; affine uses 6).
template <bool PERSPECTIVE, bool BILINEAR>
int launch_warp_stream(cudaStream_t s, const float* src, float* dst, uint32_t sw, uint32_t sh, uint32_t dw, uint32_t dh, uint32_t batch,
                       const float* minv, bool* handled) {
    *handled = false;
    if ((sw & 3u) || !aligned16(src) || sw < 16u || sh < 2u) return KB200_OK;   // TMA row copies need 16-byte aligned rows
    auto map = [&](double x, double y, double* sx, double* sy) -> bool {
        double w = 1.0;
        if (PERSPECTIVE) w = (double)minv[6] * x + (double)minv[7] * y + (double)minv[8];
        if (!(std::fabs(w) > 1e-6)) return false;
        *sx = ((double)minv[0] * x + (double)minv[1] * y + (double)minv[2]) / w;
        *sy = ((double)minv[3] * x + (double)minv[4] * y + (double)minv[5]) / w;
        return std::isfinite(*sx) && std::isfinite(*sy);
    };
    // Gentleness of the map, sampled on a 5 x 5 grid of the destination: source rows crossed by a TW-wide segment (band
    // height) and source columns covered by it (span width).  The device re-derives both per unit and falls back per tap,
    // so this only decides whether the streaming design is the FAST one here, and how large the ring must be.
    const int force = knob(KNOB_WARP_PATH);
    auto plan = [&](int npx, uint32_t* nslot_out, uint32_t* slot_out) -> bool {
        const uint32_t TW = WS_CT * (uint32_t)npx;
        double band = 0.0, span = 0.0, vstep_min = 1e30;
        for (int iy = 0; iy < 5; ++iy)
            for (int ix = 0; ix < 5; ++ix) {
                const double x = (double)(dw - 1) * ix / 4.0, y = (double)(dh - 1) * iy / 4.0;
                const double xe = std::min<double>(x + TW - 1, dw - 1);
                double ax, ay, bx, by, cx, cy;
                if (!map(x, y, &ax, &ay) || !map(xe, y, &bx, &by) || !map(x, std::min<double>(y + 1.0, dh - 1), &cx, &cy)) return false;
                const double frac = (xe > x) ? (double)(TW - 1) / (xe - x) : 1.0;   // normalise a clipped segment to a full tile
                band = std::max(band, std::fabs(by - ay) * frac);
                span = std::max(span, std::fabs(bx - ax) * frac);
                if (y + 1.0 <= dh - 1) vstep_min = std::min(vstep_min, cy - ay);
            }
        if (!(vstep_min > 0.05)) return false;      // the band must move DOWN the source (flips / 90-degree rotations: other kernels)
        uint32_t nslot = 16;
        while ((double)nslot < band + 3.0 + 6.0 && nslot < (uint32_t)WS_MAX_SLOTS) nslot <<= 1;   // band + slack + prefetch depth
        if ((double)nslot < band + 3.0 + 2.0) return false;
        const int ks = knob(KNOB_WS_STAGES);
        if (ks >= 4 && ks <= WS_MAX_SLOTS && (ks & (ks - 1)) == 0) nslot = (uint32_t)ks;
        uint32_t slot = (uint32_t)((span + 6.0) * 3.0) + 8u;
        slot = (slot + 31u) & ~31u;
        slot = std::min(slot, (sw * 3u + 31u) & ~31u);
        *nslot_out = nslot; *slot_out = slot;
        return true;
    };
    // widest tile whose ring stays small enough for several CTAs per SM; a steeper map narrows the tile first, then grows the ring
    int npx = 0;
    uint32_t nslot = 0, slot = 0;
    // bilinear: the pair-row fast consumer (warp_stream2.cu) owns one column per thread; knob ws.npx = 2 or 3 selects
    // the generic consumer instead (3 = generic with one column)
    int knpx = knob(KNOB_WS_NPX);
    const bool use_fast = BILINEAR && knpx <= 1;
    if (use_fast) knpx = 1;
    if (knpx == 3) knpx = 1;
    // default dispatch takes only GENTLE maps (ring <= 64 KB: several CTAs per SM); steeper ones go to the TMA-tiled or gather
    // kernels (warp.cu) unless the streaming path is forced (knob warp.path = 3: up to a 112 KB ring, then anything)
    for (int pass = 0; pass < (force == 3 ? 2 : 1) && npx == 0; ++pass) {
        const double cap = (pass == 0 ? 64.0 : 112.0) * 1024.0;
        for (int cand = 2; cand >= 1; --cand) {
            if (knpx >= 1 && knpx <= 2 && cand != knpx) continue;
            if (cand == 2 && dw <= 128u) continue;
            uint32_t ns, sl;
            if (plan(cand, &ns, &sl) && ((double)ns * sl * 4.0 <= cap || force == 3)) { npx = cand; nslot = ns; slot = sl; break; }
        }
    }
    if (npx == 0) return KB200_OK;
    WarpStreamParams P;
    P.sw = sw; P.sh = sh; P.dw = dw; P.dh = dh;
    for (int i = 0; i < 9; ++i) P.m[i] = (PERSPECTIVE || i < 6) ? minv[i] : 0.0f;
    P.slot_floats = slot; P.row_floats = sw * 3u; P.nslot = nslot;
    P.nslot_log2 = 0;
    while ((1u << P.nslot_log2) < nslot) ++P.nslot_log2;
    P.vec_store = ((dw & 3u) == 0 && aligned16(dst)) ? 1u : 0u;
    int per_sm = knob(KNOB_WS_CTAS) > 0 ? knob(KNOB_WS_CTAS) : 4;
    const uint32_t rc = knob(KNOB_WS_RC) > 0 ? (uint32_t)knob(KNOB_WS_RC) : 0u;
    if (use_fast) return ws2_launch<PERSPECTIVE>(s, src, dst, P, batch, knob(KNOB_WS_CTAS) > 0 ? per_sm : 8, rc, handled);
    if (npx == 1) return ws_launch<PERSPECTIVE, BILINEAR, 1>(s, src, dst, P, batch, per_sm, rc, handled);
    return ws_launch<PERSPECTIVE, BILINEAR, 2>(s, src, dst, P, batch, per_sm, rc, handled);
}

template int launch_warp_stream<false, false>(cudaStream_t, const float*, float*, uint32_t, uint32_t, uint32_t, uint32_t, uint32_t, const float*, bool*);
template int launch_warp_stream<false, true>(cudaStream_t, const float*, float*, uint32_t, uint32_t, uint32_t, uint32_t, uint32_t, const float*, bool*);
template int launch_warp_stream<true, false>(cudaStream_t, const float*, float*, uint32_t, uint32_t, uint32_t, uint32_t, uint32_t, const float*, bool*);
template int launch_warp_stream<true, true>(cudaStream_t, const float*, float*, uint32_t, uint32_t, uint32_t, uint32_t, uint32_t, const float*, bool*);

}  // namespace kb200
