// warp_stream.cuh — shared pieces of the row-streaming warp kernels (warp_stream.cu: generic consumer, any sampler;
// warp_stream2.cu: the bilinear fast consumer).  See warp_stream.cu for the design.
#pragma once

#include "kb200_common.cuh"
#include "tma_ring.cuh"
#include "warp_common.cuh"

namespace kb200 {

static constexpr int WS_CT = 128;
static constexpr int WS_THREADS = WS_CT + 32;
static constexpr int WS_MAX_SLOTS = 64;

struct WarpStreamParams {
    uint32_t sw, sh, dw, dh;
    float m[9];
    uint32_t tiles_x, chunks_y, rows_per_chunk, nunits;
    uint32_t slot_floats;     // floats per ring slot (multiple of 32)
    uint32_t row_floats;      // sw * 3
    uint32_t nslot;           // power of two
    uint32_t nslot_log2;
    uint32_t vec_store;       // destination rows are 16-byte aligned (dw % 4 == 0, aligned base)
    uint32_t dtx, dcy, dimg;
};

// approximate inverse map (schedule / span planning only — results never depend on it)
template <bool PERSPECTIVE>
__device__ __forceinline__ bool ws_plan_coord(const float* __restrict__ m, float x, float y, float* sx, float* sy) {
    if (PERSPECTIVE) {
        const float w = m[6] * x + m[7] * y + m[8];
        if (!(fabsf(w) > 1e-6f)) return false;
        const float r = 1.0f / w;
        *sx = (m[0] * x + m[1] * y + m[2]) * r;
        *sy = (m[3] * x + m[4] * y + m[5]) * r;
    } else {
        *sx = m[0] * x + (m[1] * y + m[2]);
        *sy = m[3] * x + (m[4] * y + m[5]);
    }
    return fabsf(*sx) < 1.0e8f && fabsf(*sy) < 1.0e8f;
}

// Column span [c0, c1) (floats, 4-float aligned) of the source a unit may tap: bounding box of the unit's four corners
// (exact for a projective map with a same-signed denominator), +-1 px, the +1 tap; clipped to the row and to one slot.
template <bool PERSPECTIVE>
__device__ __forceinline__ void ws_span(const WarpStreamParams& P, uint32_t dx0, uint32_t dx1, uint32_t y0, uint32_t y1, int* c0, int* c1) {
    float mn = 3.0e38f, mx = -3.0e38f;
    bool ok = true;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        float sx, sy;
        ok = ws_plan_coord<PERSPECTIVE>(P.m, (float)((k & 1) ? dx1 : dx0), (float)((k & 2) ? y1 : y0), &sx, &sy) && ok;
        mn = fminf(mn, sx); mx = fmaxf(mx, sx);
    }
    if (!ok) { *c0 = 0; *c1 = 0; return; }
    int a = ((int)floorf(mn) - 1) * 3, b = ((int)floorf(mx) + 3) * 3;
    a = max(a, 0) & ~3;
    b = min((b + 3) & ~3, (int)P.row_floats);
    if (b - a > (int)P.slot_floats) b = a + (int)P.slot_floats;   // wider than a slot: the right part falls back to global loads
    if (b < a) b = a;
    *c0 = a; *c1 = b;
}

// Schedule of 32 destination rows (lane = row): rows [lo, hi] of the source are needed by destination row dy0 + lane of the
// column segment [dx0, dx1].  Returns through lo/hi (lo > hi: nothing needed).
template <bool PERSPECTIVE>
__device__ __forceinline__ void ws_row_need(const WarpStreamParams& P, uint32_t dx0, uint32_t dx1, uint32_t dy, bool active, int* lo, int* hi) {
    *lo = 1; *hi = 0;
    if (!active) return;
    float ax, ay, bx, by;
    if (!ws_plan_coord<PERSPECTIVE>(P.m, (float)dx0, (float)dy, &ax, &ay)) return;
    if (!ws_plan_coord<PERSPECTIVE>(P.m, (float)dx1, (float)dy, &bx, &by)) return;
    const float mn = fminf(ay, by), mx = fmaxf(ay, by);
    if (mx < -1.0f || mn > (float)P.sh) return;
    int l = (int)floorf(mn) - 1, h = (int)floorf(mx) + 2;   // +-1 row of slack for the rounding of the exact coordinates, +1 tap
    l = max(l, 0); h = min(h, (int)P.sh - 1);
    if (l <= h) { *lo = l; *hi = h; }
}

// Per 32-row block, every warp derives the same two monotone row pointers (absolute source rows):
//   rel[i]: rows < rel may be dropped before destination row i is processed,
//   ld[i] : rows <= ld are resident before destination row i is processed (capped so that ld - rel < nslot).
// `rel_in` / `ld_in` carry the pointers across blocks (ld_in = last loaded row, rel_in = first not yet released row).
__device__ __forceinline__ void ws_schedule(int lo, int hi, int rel_in, int ld_in, int nslot, int* rel, int* ld) {
    const uint32_t lane = threadIdx.x & 31u;
    // suffix minimum of lo over the block's non-empty rows (a later row of the block may still need an early source row)
    int smin = (lo <= hi) ? lo : 0x7FFFFFFF;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int v = __shfl_down_sync(0xFFFFFFFFu, smin, o);
        if (lane + o < 32u) smin = min(smin, v);
    }
    // prefix maximum, carried in: pointers never move backwards
    int r = (smin == 0x7FFFFFFF) ? rel_in : max(smin, rel_in);
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int v = __shfl_up_sync(0xFFFFFFFFu, r, o);
        if (lane >= (uint32_t)o) r = max(r, v);
    }
    int l = (lo <= hi) ? max(hi, ld_in) : ld_in;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int v = __shfl_up_sync(0xFFFFFFFFu, l, o);
        if (lane >= (uint32_t)o) l = max(l, v);
    }
    // release never passes what is loaded + 1; loading never runs more than a ring ahead of the release pointer (both stay
    // monotone: the minimum of two non-decreasing sequences is non-decreasing)
    r = min(r, l + 1);
    l = min(l, r + nslot - 1);
    *rel = r; *ld = l;
}


// Need of a PAIR of destination rows (2k, 2k+1 of the block): both lanes of the pair carry the union, so a consumer that
// processes two rows per step sees one (rel, ld) for the pair and the ring-capacity cap holds for the pair as a whole.
__device__ __forceinline__ void ws_pair_need(int* lo, int* hi) {
    const int lo2 = __shfl_xor_sync(0xFFFFFFFFu, *lo, 1), hi2 = __shfl_xor_sync(0xFFFFFFFFu, *hi, 1);
    const bool a = *lo <= *hi, b = lo2 <= hi2;
    if (a && b) { *lo = min(*lo, lo2); *hi = max(*hi, hi2); }
    else if (b) { *lo = lo2; *hi = hi2; }
}

// The producer warp of a streaming kernel: all lanes compute the schedule, lane 0 issues the copies.
template <bool PERSPECTIVE, bool PAIR, uint32_t TW>
__device__ __forceinline__ void ws_producer(const float* __restrict__ src, const WarpStreamParams& P, float* ring, uint64_t* full_bar,
                                            uint64_t* empty_bar) {
    const uint32_t lane = threadIdx.x & 31u;
    const int nslot = (int)P.nslot;
    const uint32_t smask = P.nslot - 1u;
    const size_t src_img = (size_t)P.row_floats * P.sh;
    tma::UnitWalk<WarpStreamParams> w;
    w.init(blockIdx.x, P);
    uint32_t qbase = 0;
    for (uint32_t u = blockIdx.x; u < P.nunits; u += gridDim.x, w.advance(P)) {
        const uint32_t dx0 = w.tx * TW, dx1 = min(dx0 + TW, P.dw) - 1u;
        const uint32_t y_first = w.cy * P.rows_per_chunk, y_end = min(y_first + P.rows_per_chunk, P.dh);
        int c0, c1;
        ws_span<PERSPECTIVE>(P, dx0, dx1, y_first, y_end - 1u, &c0, &c1);
        const uint32_t bytes = (uint32_t)(c1 - c0) * 4u;
        const float* frame = src + (size_t)w.img * src_img + c0;
        int r0 = -1, rel_c = 0, ld_c = -1;   // r0: first resident row of the unit (set by the first non-empty block)
        for (uint32_t yb = y_first; yb < y_end; yb += 32u) {
            int lo, hi;
            ws_row_need<PERSPECTIVE>(P, dx0, dx1, yb + lane, yb + lane < y_end, &lo, &hi);
            if (PAIR) ws_pair_need(&lo, &hi);
            if (r0 < 0) {   // anchor the unit at the first needed row (warp-uniform)
                int first = (lo <= hi) ? lo : 0x7FFFFFFF;
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) first = min(first, __shfl_xor_sync(0xFFFFFFFFu, first, o));
                if (first == 0x7FFFFFFF) continue;   // nothing needed by this block
                r0 = first; rel_c = first; ld_c = first - 1;
            }
            int rel, ld;
            ws_schedule(lo, hi, rel_c, ld_c, nslot, &rel, &ld);
            const int ld_last = __shfl_sync(0xFFFFFFFFu, ld, 31), rel_last = __shfl_sync(0xFFFFFFFFu, rel, 31);
            if (lane == 0 && bytes != 0u) {
                // rows ld_c+1 .. ld_last in order; each waits only for its own slot (released in order by the consumers)
                for (int r = ld_c + 1; r <= ld_last; ++r) {
                    const uint32_t q = qbase + (uint32_t)(r - r0);
                    const uint32_t slot = q & smask, use = q >> P.nslot_log2;
                    if (use > 0) tma::mbar_wait_backoff(&empty_bar[slot], (use - 1u) & 1u);
                    tma::mbar_expect_tx(&full_bar[slot], bytes);
                    tma::load_1d(ring + (size_t)slot * P.slot_floats, frame + (size_t)r * P.row_floats, bytes, &full_bar[slot]);
                }
            }
            rel_c = rel_last; ld_c = ld_last;
        }
        if (r0 >= 0 && bytes != 0u) qbase += (uint32_t)(ld_c - r0 + 1);
    }
}

}  // namespace kb200
