// filter_u8.cu — u8 blurs (SURVEY §8(f) #1): gaussian_blur_u8 / box_blur_u8.
//
// Reference: filter/ops.rs:22-29 (blur_u8_path), :59-98 (box_blur_u8), :639-757 (gaussian_blur_u8), :759-770
// (quantize_kernel_256), :773-851 + :852-1100 (general Q8 two-pass: H pass (acc + 128) >> 8 into a u8 intermediate with
// the row replicated left/right, V pass likewise over row-clamped H rows), :1105-1285 (k = 3, sigma in [0.6, 1.2]:
// [1,2,1]/4 as rhadd(rhadd(a,b), rhadd(b,d)) per axis).  Integer arithmetic throughout — bit-exact class.
//
// Kernel: one CTA per (image, 32x32-pixel tile).  The tile plus its halo is gathered into shared memory with the
// replicate rule applied at gather time, the H pass writes its u8 result to a second shared array (the reference's u8
// intermediate — the rounding between the passes is part of the result), the V pass reads it and stores.  Both the
// Q8 and the binomial arithmetic run through the same staging.
#include <algorithm>
#include <vector>

#include "kb200_common.cuh"
#include "tma_ring.cuh"

namespace kb200 {

static constexpr int U8B_TW = 32, U8B_TH = 32, U8B_MAXK = 31;

struct U8Taps {
    uint8_t kx[32], ky[32];
    int kxn, kyn;
    int binomial;   // 1: [1,2,1]/4 rounding half-add path (kxn = kyn = 3)
};

__device__ __forceinline__ uint32_t rhadd_u8(uint32_t a, uint32_t b) { return (a + b + 1u) >> 1; }

// K > 0: both axes have K taps, held in registers (the loops unroll); K == 0: run-time tap counts, taps read from shared
// memory.  (Indexing the taps in the kernel-parameter bank costs one LDC per tap per byte — measured 5x slower.)
template <int C, int K>
__global__ void __launch_bounds__(256) blur_u8_tile_kernel(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst, uint32_t cols,
                                                           uint32_t rows, uint32_t tiles_x, uint32_t tiles_y,
                                                           const __grid_constant__ U8Taps T) {
    extern __shared__ uint8_t u8b_smem[];
    __shared__ uint32_t tap_s[2][32];
    const int kxn = K > 0 ? K : T.kxn, kyn = K > 0 ? K : T.kyn;
    uint32_t kxr[K > 0 ? K : 1], kyr[K > 0 ? K : 1];
    if (K > 0) {
#pragma unroll
        for (int k = 0; k < (K > 0 ? K : 1); ++k) { kxr[k] = T.kx[k]; kyr[k] = T.ky[k]; }
    } else if (threadIdx.x < 32) {
        tap_s[0][threadIdx.x] = T.kx[threadIdx.x]; tap_s[1][threadIdx.x] = T.ky[threadIdx.x];
    }
    const int hx = kxn / 2, hy = kyn / 2;
    const int in_wpx = U8B_TW + 2 * hx, in_h = U8B_TH + 2 * hy;
    const int in_wb = in_wpx * C, mid_wb = U8B_TW * C;
    uint8_t* in = u8b_smem;                       // [in_h][in_wb]
    uint8_t* mid = u8b_smem + (size_t)in_h * in_wb;   // [in_h][mid_wb]
    const uint32_t t = blockIdx.x;
    const uint32_t img = t / (tiles_x * tiles_y), tt = t - img * tiles_x * tiles_y;
    const int x0 = (int)(tt % tiles_x) * U8B_TW, y0 = (int)(tt / tiles_x) * U8B_TH;
    const uint8_t* s = src + (size_t)img * cols * rows * C;
    uint8_t* d = dst + (size_t)img * cols * rows * C;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;   // 32 x 8: rows by ty, bytes / pixels by tx — no index divisions
    // gather with the replicate rule (clamped row / column indices)
    for (int r = ty; r < in_h; r += 8) {
        const int sy = min(max(y0 - hy + r, 0), (int)rows - 1);
        const uint8_t* srow = s + (size_t)sy * cols * C;
        for (int p = tx; p < in_wpx; p += 32) {
            const int sx = min(max(x0 - hx + p, 0), (int)cols - 1);
#pragma unroll
            for (int ch = 0; ch < C; ++ch) in[r * in_wb + p * C + ch] = srow[sx * C + ch];
        }
    }
    __syncthreads();
    // H pass -> u8 intermediate
    for (int r = ty; r < in_h; r += 8) {
        for (int j = tx; j < mid_wb; j += 32) {
            const uint8_t* ip = in + r * in_wb + j;          // tap k at ip[k*C]
            uint32_t v;
            if (T.binomial) v = rhadd_u8(rhadd_u8(ip[0], ip[C]), rhadd_u8(ip[C], ip[2 * C]));
            else {
                uint32_t acc = 0;
                if (K > 0) {
#pragma unroll
                    for (int k = 0; k < (K > 0 ? K : 1); ++k) acc += (uint32_t)ip[k * C] * kxr[k];
                } else {
                    for (int k = 0; k < kxn; ++k) acc += (uint32_t)ip[k * C] * tap_s[0][k];
                }
                v = (acc + 128u) >> 8;
            }
            mid[r * mid_wb + j] = (uint8_t)v;
        }
    }
    __syncthreads();
    // V pass -> global
    for (int r = ty; r < U8B_TH; r += 8) {
        const int gy = y0 + r;
        if (gy >= (int)rows) break;
        uint8_t* drow = d + (size_t)gy * cols * C + (size_t)x0 * C;
        const int nb = min(mid_wb, ((int)cols - x0) * C);
        for (int j = tx; j < nb; j += 32) {
            const uint8_t* mp = mid + r * mid_wb + j;        // tap k at mp[k*mid_wb]
            uint32_t v;
            if (T.binomial) v = rhadd_u8(rhadd_u8(mp[0], mp[mid_wb]), rhadd_u8(mp[mid_wb], mp[2 * mid_wb]));
            else {
                uint32_t acc = 0;
                if (K > 0) {
#pragma unroll
                    for (int k = 0; k < (K > 0 ? K : 1); ++k) acc += (uint32_t)mp[k * mid_wb] * kyr[k];
                } else {
                    for (int k = 0; k < kyn; ++k) acc += (uint32_t)mp[k * mid_wb] * tap_s[1][k];
                }
                v = (acc + 128u) >> 8;
            }
            drow[j] = (uint8_t)v;
        }
    }
}

// ── word-granular variant ────────────────────────────────────────────────────────────────────
// ncu-free arithmetic on the kernel above: ~15 LSU operations per output byte (byte gathers, one LDS.U8 per tap per
// byte, byte stores) against 1.5 B of DRAM traffic per byte — LSU-bound, far below the roofline.  Here every access is
// a 32-bit word and four bytes are filtered at once in two 16-bit lanes per register:
//   e = w & 0x00FF00FF, o = (w >> 8) & 0x00FF00FF;  acc_e += e * k, acc_o += o * k
// A lane never overflows: Σ byte·k <= 255 · Σk = 255 · 256 < 2^16 (the host checks Σk <= 256), and the Q8 rounding
// (+128, >> 8) is applied per lane, so each byte gets exactly the reference's u32 arithmetic.  The binomial path is
// the per-byte rounded average (a | b) - (((a ^ b) >> 1) & 0x7F7F7F7F) == (a + b + 1) >> 1.
// The staged tile keeps the global word alignment of its first byte: tile byte j lives at shared byte j + SH0 with
// SH0 = (-(K/2)*C) mod 4 (a tile starts at a multiple of 32 pixels), so interior tiles are gathered with aligned
// LDG.32 / STS.32 and a tap's four bytes are one funnel shift of two neighbouring words at a compile-time offset.
// Needs cols*C % 4 == 0 and 4-byte aligned images; anything else uses the byte kernel.
__device__ __forceinline__ uint32_t avg4_round_up(uint32_t a, uint32_t b) { return (a | b) - (((a ^ b) >> 1) & 0x7F7F7F7Fu); }

static constexpr int U8W_TW = 64, U8W_TH = 64;   // word kernel: larger tiles amortise the two block-wide phase changes and the halo rows

template <int C, int K>
__global__ void __launch_bounds__(256) blur_u8_tile_w_kernel(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst, uint32_t cols,
                                                             uint32_t rows, uint32_t tiles_x, uint32_t tiles_y,
                                                             const __grid_constant__ U8Taps T) {
    constexpr int HX = K / 2, HY = K / 2;
    constexpr int SH0 = ((-(HX * C)) % 4 + 4) % 4;
    constexpr int IN_WPX = U8W_TW + 2 * HX, IN_H = U8W_TH + 2 * HY;
    constexpr int IN_WW = (IN_WPX * C + SH0 + 3) / 4 + 1;        // words per staged row (+1: the last funnel shift reads one word further)
    constexpr int MID_WW = U8W_TW * C / 4;                       // words per intermediate row
    constexpr int NW = (SH0 + (K - 1) * C + 4 + 3) / 4 + 1;      // words covering all taps of one 4-byte output
    extern __shared__ uint32_t u8w_smem[];
    uint32_t* in = u8w_smem;                                     // [IN_H][IN_WW]
    uint32_t* mid = u8w_smem + IN_H * IN_WW;                     // [IN_H][MID_WW]
    uint32_t kx[K], ky[K];
#pragma unroll
    for (int k = 0; k < K; ++k) { kx[k] = T.kx[k]; ky[k] = T.ky[k]; }
    const bool binomial = T.binomial != 0;
    const uint32_t t = blockIdx.x;
    const uint32_t img = t / (tiles_x * tiles_y), tt = t - img * tiles_x * tiles_y;
    const int x0 = (int)(tt % tiles_x) * U8W_TW, y0 = (int)(tt / tiles_x) * U8W_TH;
    const uint32_t rowb = cols * C;                              // bytes per image row, multiple of 4
    const uint8_t* s = src + (size_t)img * rowb * rows;
    uint8_t* d = dst + (size_t)img * rowb * rows;
    const int tid = threadIdx.x, tx = tid & 31, ty = tid >> 5;
    const bool interior_x = x0 - HX >= 0 && x0 + U8W_TW + HX <= (int)cols;
    // ── gather (rows clamped; columns clamped only on edge tiles) ──
    if (interior_x) {
        const int abase = (x0 - HX) * C - SH0;                   // global byte of shared word 0: multiple of 4, >= -3
        for (int r = ty; r < IN_H; r += 8) {
            const int sy = min(max(y0 - HY + r, 0), (int)rows - 1);
            const uint32_t* srow = reinterpret_cast<const uint32_t*>(s + (size_t)sy * rowb);
            for (int w = tx; w < IN_WW; w += 32) {
                const int gb = abase + 4 * w;                    // first global byte of this word
                // the first word may start before the row (SH0 bytes of slack) and the last may end after it: those
                // bytes are never used by a tap, so any in-bounds word will do
                const int gw = min(max(gb, 0), (int)rowb - 4) >> 2;
                in[r * IN_WW + w] = __ldg(srow + gw);
            }
        }
    } else {
        uint8_t* inb = reinterpret_cast<uint8_t*>(in);
        for (int r = ty; r < IN_H; r += 8) {
            const int sy = min(max(y0 - HY + r, 0), (int)rows - 1);
            const uint8_t* srow = s + (size_t)sy * rowb;
            for (int p = tx; p < IN_WPX; p += 32) {
                const int sx = min(max(x0 - HX + p, 0), (int)cols - 1);
#pragma unroll
                for (int ch = 0; ch < C; ++ch) inb[r * IN_WW * 4 + SH0 + p * C + ch] = srow[sx * C + ch];
            }
        }
    }
    __syncthreads();
    // ── H pass: 4 output bytes per item ──
    for (int i = tid; i < IN_H * MID_WW; i += 256) {
        const int r = i / MID_WW, q = i - r * MID_WW;
        const uint32_t* ip = in + r * IN_WW + q;
        uint32_t W[NW];
#pragma unroll
        for (int n = 0; n < NW; ++n) W[n] = ip[n];
        uint32_t v;
        if (binomial) {
            uint32_t x[3];
#pragma unroll
            for (int k = 0; k < 3; ++k) { constexpr int dummy = 0; (void)dummy; const int off = SH0 + k * C; x[k] = __funnelshift_r(W[off >> 2], W[(off >> 2) + 1], 8 * (off & 3)); }
            v = avg4_round_up(avg4_round_up(x[0], x[1]), avg4_round_up(x[1], x[2]));
        } else {
            uint32_t ae = 0x00800080u, ao = 0x00800080u;         // + 128 per lane
#pragma unroll
            for (int k = 0; k < K; ++k) {
                const int off = SH0 + k * C;
                const uint32_t x = __funnelshift_r(W[off >> 2], W[(off >> 2) + 1], 8 * (off & 3));
                ae += (x & 0x00FF00FFu) * kx[k];
                ao += ((x >> 8) & 0x00FF00FFu) * kx[k];
            }
            v = ((ae >> 8) & 0x00FF00FFu) | (ao & 0xFF00FF00u);
        }
        mid[r * MID_WW + q] = v;
    }
    __syncthreads();
    // ── V pass -> global words ──
    const int nwords = min(MID_WW, (int)((cols - (uint32_t)x0) * C / 4));   // valid words of this tile row
    for (int i = tid; i < U8W_TH * MID_WW; i += 256) {
        const int r = i / MID_WW, q = i - r * MID_WW;
        const int gy = y0 + r;
        if (gy >= (int)rows || q >= nwords) continue;
        const uint32_t* mp = mid + r * MID_WW + q;
        uint32_t v;
        if (binomial) v = avg4_round_up(avg4_round_up(mp[0], mp[MID_WW]), avg4_round_up(mp[MID_WW], mp[2 * MID_WW]));
        else {
            uint32_t ae = 0x00800080u, ao = 0x00800080u;
#pragma unroll
            for (int k = 0; k < K; ++k) {
                const uint32_t x = mp[k * MID_WW];
                ae += (x & 0x00FF00FFu) * ky[k];
                ao += ((x >> 8) & 0x00FF00FFu) * ky[k];
            }
            v = ((ae >> 8) & 0x00FF00FFu) | (ao & 0xFF00FF00u);
        }
        reinterpret_cast<uint32_t*>(d + (size_t)gy * rowb + (size_t)x0 * C)[q] = v;
    }
}

// ── row-streaming variant (round 2) ───────────────────────────────────────────────────────────
// The tile kernel above pays two block-wide phase changes, a (64+K-1)^2 / 64^2 halo and a shared-memory round trip of the
// intermediate per tile.  This is the u8 twin of sep_filter_stream2 (filter.cu): a unit is
// (image, strip of 128*NV words of a row, chunk of rows); every source row span is copied ONCE global -> shared by the
// TMA engine (tma::load_1d, mbarrier ring, producer lane; rows clamped = the reference's replicate border in y); a
// consumer thread owns NV word columns: the H pass reads the words around its column (compile-time funnel shifts per tap,
// two 16-bit lanes per register as above), its result goes — split into even and odd bytes — into a K-deep rotating REGISTER
// window, and as soon as the window is full the V pass emits one lane-contiguous STG.32 per column.  The u8 intermediate never
// leaves registers; no __syncthreads in the loop.  The replicate border in x is a 16-byte halo patch in shared memory (below).
// Needs rows of a multiple of 16 bytes and 16-byte aligned images (TMA); anything else uses the tile kernels.
static constexpr int U8S_CT = 128, U8S_THREADS = U8S_CT + 32, U8S_MAX_STAGES = 16, U8S_HALO = 16;

struct U8StreamParams {
    uint32_t rowb, rows, strips, chunks, rows_per_chunk, nunits, stages, slot_bytes;
};

// Replicate border in x without an edge path: after a row has landed, the warp that owns the first word of the row writes
// the 16 halo bytes left of it (bytes at row position p < 0 are channel p mod C of pixel 0 — a byte permutation of the row's
// first word), and the warp that owns the last word writes the 16 bytes right of it (channel q mod C of the last pixel — a
// permutation of the last word; rows are a multiple of 16 bytes, so the four words around the row end sit in one warp).  Both
// regions are outside what the TMA copy writes.  Every thread then takes the same word-granular taps.  (Round 2 had a byte-wise
// clamped path for the threads at the border: inlined it cost 127 registers and an instruction-cache-missing kernel, out of
// line it stalled the whole CTA behind one warp.)
template <int C>
__host__ __device__ constexpr uint32_t u8s_sel_left(int j) {          // word j of the halo: row positions -16 + 4j .. + 3
    uint32_t sel = 0;
    for (int b = 0; b < 4; ++b) { const int p = -16 + 4 * j + b; sel |= (uint32_t)(((p % C) + C) % C) << (4 * b); }
    return sel;
}
template <int C>
__host__ __device__ constexpr uint32_t u8s_sel_right(int j) {         // word j past the row end: row positions rowb + 4j .. + 3
    uint32_t sel = 0;
    for (int b = 0; b < 4; ++b) { const int q = 4 * j + b; sel |= (uint32_t)(4 - C + (q % C)) << (4 * b); }
    return sel;
}

template <int C, int K, int NV>
__global__ void __launch_bounds__(U8S_THREADS) blur_u8_stream_kernel(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst,
                                                                     const __grid_constant__ U8Taps T, const __grid_constant__ U8StreamParams P) {
    constexpr int HX = K / 2, HY = K / 2;
    constexpr int EB = U8S_CT * NV * 4;                       // bytes of a strip
    static_assert(HX * C <= U8S_HALO, "halo");
    extern __shared__ __align__(128) uint8_t u8s_smem[];
    __shared__ __align__(8) uint64_t full_bar[U8S_MAX_STAGES];
    __shared__ __align__(8) uint64_t empty_bar[U8S_MAX_STAGES];
    const uint32_t tid = threadIdx.x, nst = P.stages;
    if (tid == 0) {
        for (uint32_t s = 0; s < nst; ++s) { tma::mbar_init(&full_bar[s], 1); tma::mbar_init(&empty_bar[s], U8S_CT / 32); }
        tma::mbar_fence_init();
    }
    __syncthreads();
    const size_t img_bytes = (size_t)P.rowb * P.rows;
    uint32_t stage = 0, phase = 0;

    if (tid >= U8S_CT) {
        if (tid != U8S_CT) return;
        bool first_lap = true;
        for (uint32_t u = blockIdx.x; u < P.nunits; u += gridDim.x) {
            const uint32_t strip = u % P.strips, rest = u / P.strips;
            const uint32_t chunk = rest % P.chunks, img = rest / P.chunks;
            const int e0 = (int)(strip * EB);
            const int g0 = max(e0 - U8S_HALO, 0), g1 = min(e0 + EB + U8S_HALO, (int)P.rowb);   // multiples of 16
            const uint32_t bytes = (uint32_t)(g1 - g0);
            const uint32_t slot_off = (uint32_t)(g0 - (e0 - U8S_HALO));
            const int y_first = (int)(chunk * P.rows_per_chunk), y_end = min(y_first + (int)P.rows_per_chunk, (int)P.rows);
            const uint8_t* base = src + (size_t)img * img_bytes + g0;
            for (int iy = y_first - HY; iy < y_end + HY; ++iy) {
                if (!first_lap) tma::mbar_wait(&empty_bar[stage], phase ^ 1u);
                const int sy = min(max(iy, 0), (int)P.rows - 1);          // replicate border in y: the clamped row (filter/ops.rs:852-1100)
                tma::mbar_expect_tx(&full_bar[stage], bytes);
                tma::load_1d(u8s_smem + (size_t)stage * P.slot_bytes + slot_off, base + (size_t)sy * P.rowb, bytes, &full_bar[stage]);
                if (++stage == nst) { stage = 0; phase ^= 1u; first_lap = false; }
            }
        }
        return;
    }

    uint32_t kx[7], ky[7];
#pragma unroll
    for (int k = 0; k < 7; ++k) { kx[k] = k < K ? T.kx[k] : 0u; ky[k] = k < K ? T.ky[k] : 0u; }
    const bool binomial = K == 3 && T.binomial != 0;
    const bool lane0 = (tid & 31u) == 0;
    const int cols = (int)(P.rowb / C);
    for (uint32_t u = blockIdx.x; u < P.nunits; u += gridDim.x) {
        const uint32_t strip = u % P.strips, rest = u / P.strips;
        const uint32_t chunk = rest % P.chunks, img = rest / P.chunks;
        const int e0 = (int)(strip * EB);
        const int y_first = (int)(chunk * P.rows_per_chunk), y_end = min(y_first + (int)P.rows_per_chunk, (int)P.rows);
        uint8_t* out = dst + (size_t)img * img_bytes + (size_t)y_first * P.rowb;
        int B[NV];            // first global byte (within the row) of this thread's word column v
        bool act[NV];
#pragma unroll
        for (int v = 0; v < NV; ++v) {
            B[v] = e0 + 4 * ((int)tid + v * U8S_CT);
            act[v] = B[v] < (int)P.rowb;
        }
        const int last_word = ((int)P.rowb - e0) / 4 - 1;                                   // strip-relative word index of the row's last word
        const bool lpatch = e0 == 0 && tid < 32u;                                          // this warp owns the row's first word
        const bool rpatch = last_word < U8S_CT * NV && ((last_word % U8S_CT) >> 5) == (int)(tid >> 5);   // ... its last word (warp-uniform)
        // K-deep register window of H-pass results, oldest first.  The row loop is NOT unrolled: rotating the window costs
        // (K-1)*NV register moves per row, whereas K unrolled copies of the row step made the kernel ~40 KB of code that
        // missed the instruction cache on every lap (ncu: no-instruction stalls).
        // Q8 path: the window keeps each H result SPLIT into its even and odd bytes (two 16-bit lanes per register: exactly the
        // operand form of the V pass), so the V pass is ten IMADs and one PRMT per word — no byte extraction (the kernel is bound
        // by the ALU pipe: LOP / PRMT / SHF).  The binomial path (K = 3) keeps packed bytes in win alone.
        uint32_t win[K][NV], wodd[K][NV];
#pragma unroll
        for (int s = 0; s < K; ++s)
#pragma unroll
            for (int v = 0; v < NV; ++v) { win[s][v] = 0u; wodd[s][v] = 0u; }
        const int iy_end = y_end + HY;
#pragma unroll 1
        for (int iy = y_first - HY; iy < iy_end; ++iy) {
            tma::mbar_wait(&full_bar[stage], phase);
            uint8_t* slot = u8s_smem + (size_t)stage * P.slot_bytes;                // slot byte j = row byte e0 - 16 + j
            if (lpatch) {
                if (tid == 0) {
                    uint32_t* sw = reinterpret_cast<uint32_t*>(slot);
                    const uint32_t w = sw[U8S_HALO / 4];
#pragma unroll
                    for (int j = 0; j < 4; ++j) sw[j] = __byte_perm(w, 0u, u8s_sel_left<C>(j));
                    tma::fence_proxy_async();      // a later TMA copy (another strip's row) may overwrite these bytes
                }
                __syncwarp();
            }
            if (rpatch) {
                if ((int)tid == last_word % U8S_CT) {
                    uint32_t* sw = reinterpret_cast<uint32_t*>(slot) + U8S_HALO / 4 + last_word;
                    const uint32_t w = sw[0];
#pragma unroll
                    for (int j = 0; j < 4; ++j) sw[1 + j] = __byte_perm(w, 0u, u8s_sel_right<C>(j));
                    tma::fence_proxy_async();
                }
                __syncwarp();
            }
            uint32_t hres[NV], hodd[NV];
#pragma unroll
            for (int v = 0; v < NV; ++v) {
                hres[v] = 0; hodd[v] = 0;
                if (act[v]) {
                    uint32_t x[7];
                    // tap t of output bytes B..B+3 starts at row byte B + (t - HX)*C: word index and shift are compile-time
                    // relative to this thread's word
                    const uint32_t* wp = reinterpret_cast<const uint32_t*>(slot) + (U8S_HALO / 4) + tid + v * U8S_CT;
#pragma unroll
                    for (int t = 0; t < 7; ++t) {
                        if (t >= K) break;
                        const int off = (t - HX) * C;                           // byte offset, may be negative
                        const int wi = (off >= 0) ? (off >> 2) : -((-off + 3) >> 2);
                        const int sh = off - 4 * wi;                            // 0..3
                        x[t] = sh == 0 ? wp[wi] : __funnelshift_r(wp[wi], wp[wi + 1], 8 * sh);
                    }
                    if (binomial) hres[v] = avg4_round_up(avg4_round_up(x[0], x[1]), avg4_round_up(x[1], x[2]));
                    else {
                        uint32_t ae = 0x00800080u, ao = 0x00800080u;         // + 128 per 16-bit lane
#pragma unroll
                        for (int t = 0; t < 7; ++t) {
                            if (t >= K) break;
                            ae += (x[t] & 0x00FF00FFu) * kx[t];
                            ao += __byte_perm(x[t], 0u, 0x4341u) * kx[t];
                        }
                        hres[v] = __byte_perm(ae, 0u, 0x4341u);              // (ae >> 8) & 0x00FF00FF: result bytes 0 and 2
                        hodd[v] = __byte_perm(ao, 0u, 0x4341u);              // result bytes 1 and 3
                    }
                }
            }
            __syncwarp();
            if (lane0) tma::mbar_arrive(&empty_bar[stage]);
            if (++stage == nst) { stage = 0; phase ^= 1u; }
#pragma unroll
            for (int v = 0; v < NV; ++v) {
#pragma unroll
                for (int s = 0; s + 1 < K; ++s) { win[s][v] = win[s + 1][v]; wodd[s][v] = wodd[s + 1][v]; }
                win[K - 1][v] = hres[v]; wodd[K - 1][v] = hodd[v];
            }
            // output row r = iy - HY is complete: its window is win[0..K-1]
            if (iy - HY >= y_first) {
#pragma unroll
                for (int v = 0; v < NV; ++v) {
                    if (!act[v]) continue;
                    uint32_t o;
                    if (binomial) o = avg4_round_up(avg4_round_up(win[0][v], win[1][v]), avg4_round_up(win[1][v], win[K > 2 ? 2 : 0][v]));
                    else {
                        uint32_t ve = 0x00800080u, vo = 0x00800080u;
#pragma unroll
                        for (int t = 0; t < K; ++t) { ve += win[t][v] * ky[t]; vo += wodd[t][v] * ky[t]; }
                        o = __byte_perm(ve, vo, 0x7351u);                    // high byte of each lane, even / odd interleaved
                    }
                    *reinterpret_cast<uint32_t*>(out + B[v]) = o;
                }
                out += P.rowb;
            }
        }
    }
}

template <int C, int K>
static int launch_blur_u8_stream(cudaStream_t s, const uint8_t* src, uint8_t* dst, uint32_t cols, uint32_t rows, uint32_t batch, const U8Taps& T) {
    constexpr int NV = 2;
    auto kern = blur_u8_stream_kernel<C, K, NV>;
    U8StreamParams P;
    P.rowb = cols * C; P.rows = rows;
    const uint32_t EB = U8S_CT * NV * 4;
    P.strips = (P.rowb + EB - 1) / EB;
    P.slot_bytes = EB + 2 * U8S_HALO + 32;                  // + slack: the last funnel shift reads one word past the halo
    P.slot_bytes = (P.slot_bytes + 127u) & ~127u;
    P.stages = 6;
    const size_t smem = (size_t)P.slot_bytes * P.stages;
    int resident = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&resident, kern, U8S_THREADS, smem) != cudaSuccess || resident < 1) { cudaGetLastError(); return 1; }
    const int per_sm = std::min(resident, knob(KNOB_C) > 0 ? knob(KNOB_C) : 8);
    const size_t ctas = (size_t)device_info().sm_count * per_sm;
    const size_t total = (size_t)P.strips * batch * rows;
    // rows per chunk: every chunk re-reads K-1 halo rows, so long chunks when there is enough work for ~4 units per CTA,
    // short ones otherwise
    uint32_t rc = knob(KNOB_D) > 0 ? (uint32_t)knob(KNOB_D) : (uint32_t)std::min<size_t>(128, std::max<size_t>(32, total / (ctas * 4)));
    rc = std::min(rc, rows);
    P.rows_per_chunk = rc;
    P.chunks = (rows + rc - 1) / rc;
    const size_t nunits = (size_t)P.strips * P.chunks * batch;
    if (nunits > 0x7FFFFFFFull) return 1;
    P.nunits = (uint32_t)nunits;
    kern<<<(unsigned)std::min<size_t>(nunits, ctas), U8S_THREADS, smem, s>>>(src, dst, T, P);
    return check_launch("blur_u8_stream_kernel") == KB200_OK ? 0 : -1;
}

// filter/ops.rs:759-770
static void quantize_kernel_256(const float* k, int n, uint8_t* out) {
    uint32_t sum = 0;
    for (int i = 0; i < n; ++i) {
        const float v = k[i] * 256.0f + 0.5f;
        out[i] = (v != v || v <= 0.0f) ? 0 : (v >= 255.0f ? 255 : (uint8_t)v);   // `as u8`: saturating, NaN -> 0
        sum += out[i];
    }
    if (sum != 256) {
        const int c = (int)out[n / 2] + (256 - (int)sum);
        out[n / 2] = (uint8_t)std::min(std::max(c, 0), 255);
    }
}

static int launch_blur_u8(cudaStream_t s, const uint8_t* src, size_t src_len, uint8_t* dst, size_t dst_len, uint32_t cols, uint32_t rows,
                          uint32_t C, uint32_t batch, const U8Taps& T) {
    KB200_TRY(check_ptr("src", src)); KB200_TRY(check_ptr("dst", dst));
    KB200_TRY(check_geometry(cols, rows, cols, rows, batch));
    if (!(C == 1 || C == 3 || C == 4)) return fail(KB200_ERR_UNSUPPORTED, "u8 blur supports 1, 3 or 4 channels, got %u", C);
    const size_t n = (size_t)cols * rows * C * batch;
    KB200_TRY(check_slice("src", src_len, n)); KB200_TRY(check_slice("dst", dst_len, n));
    if (src == dst) return fail(KB200_ERR_INVALID_ARGUMENT, "src and dst must not alias (tiles read a halo)");
    if ((size_t)cols * C > 0x7FFFFFFFull || rows > 0x7FFFFFFFu) return fail(KB200_ERR_DIMS_TOO_LARGE, "u8 blur image dimensions too large");
    const uint32_t tiles_x = div_up(cols, U8B_TW), tiles_y = div_up(rows, U8B_TH);
    const size_t ntiles = (size_t)tiles_x * tiles_y * batch;
    if (ntiles > 0x7FFFFFFFull) return fail(KB200_ERR_DIMS_TOO_LARGE, "too many tiles (%zu)", ntiles);
    const int hx = T.kxn / 2, hy = T.kyn / 2;
    const size_t smem = (size_t)(U8B_TH + 2 * hy) * ((U8B_TW + 2 * hx) * C + U8B_TW * C);
    auto go = [&](auto kern) -> int {
        if (smem > 40 * 1024) {
            cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
            if (e != cudaSuccess) return fail(KB200_ERR_CUDA, "cudaFuncSetAttribute(smem=%zu) failed: %s", smem, cudaGetErrorString(e));
        }
        kern<<<(unsigned)ntiles, 256, smem, s>>>(src, dst, cols, rows, tiles_x, tiles_y, T);
        return check_launch("blur_u8_tile_kernel");
    };
    // word-granular path: whole-word rows, aligned images, K in {3,5,7} on both axes, tap sums that cannot overflow a 16-bit lane
    {
        uint32_t sx = 0, sy = 0;
        for (int k = 0; k < T.kxn; ++k) sx += T.kx[k];
        for (int k = 0; k < T.kyn; ++k) sy += T.ky[k];
        const bool word_ok = ((size_t)cols * C) % 4 == 0 && ((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(dst)) & 3u) == 0 &&
                             T.kxn == T.kyn && (T.binomial || (sx <= 256 && sy <= 256)) && cols >= 4;
        // row-streaming kernel: additionally needs 16-byte rows / bases (TMA row copies) and rows long enough for a strip
        const bool stream_ok = word_ok && (T.kxn == 3 || T.kxn == 5 || T.kxn == 7) && ((size_t)cols * C) % 16 == 0 && (size_t)cols * C >= 256 &&
                               ((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(dst)) & 15u) == 0 && (T.kxn / 2) * (int)C <= U8S_HALO &&
                               knob(KNOB_B) != 3;
        if (stream_ok) {
            int r = 1;
#define KB200_U8S(CC, KK) if (C == CC && T.kxn == KK) r = launch_blur_u8_stream<CC, KK>(s, src, dst, cols, rows, batch, T);
            KB200_U8S(1, 3) KB200_U8S(1, 5) KB200_U8S(1, 7) KB200_U8S(3, 3) KB200_U8S(3, 5) KB200_U8S(3, 7) KB200_U8S(4, 3) KB200_U8S(4, 5) KB200_U8S(4, 7)
#undef KB200_U8S
            if (r == 0) return KB200_OK;
            if (r < 0) return KB200_ERR_CUDA;
        }
        if (word_ok && (T.kxn == 3 || T.kxn == 5 || T.kxn == 7)) {
            auto gow = [&](auto kern, int K) -> int {
                const int hx = K / 2;
                const int sh0 = ((-(hx * (int)C)) % 4 + 4) % 4;
                const size_t in_ww = ((U8W_TW + 2 * hx) * C + sh0 + 3) / 4 + 1, mid_ww = U8W_TW * C / 4;
                const size_t smem_w = (size_t)(U8W_TH + 2 * hx) * (in_ww + mid_ww) * 4;
                const uint32_t wtx = div_up(cols, U8W_TW), wty = div_up(rows, U8W_TH);
                const size_t wtiles = (size_t)wtx * wty * batch;
                if (smem_w > 40 * 1024) {
                    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_w);
                    if (e != cudaSuccess) return fail(KB200_ERR_CUDA, "cudaFuncSetAttribute(smem=%zu) failed: %s", smem_w, cudaGetErrorString(e));
                }
                kern<<<(unsigned)wtiles, 256, smem_w, s>>>(src, dst, cols, rows, wtx, wty, T);
                return check_launch("blur_u8_tile_w_kernel");
            };
#define KB200_U8W(CC, KK) if (C == CC && T.kxn == KK) return gow(blur_u8_tile_w_kernel<CC, KK>, KK);
            KB200_U8W(1, 3) KB200_U8W(1, 5) KB200_U8W(1, 7) KB200_U8W(3, 3) KB200_U8W(3, 5) KB200_U8W(3, 7) KB200_U8W(4, 3) KB200_U8W(4, 5) KB200_U8W(4, 7)
#undef KB200_U8W
        }
    }
#define KB200_U8B(CC)                                                                   \
    if (C == CC) {                                                                      \
        if (T.kxn == T.kyn && T.kxn == 3) return go(blur_u8_tile_kernel<CC, 3>);        \
        if (T.kxn == T.kyn && T.kxn == 5) return go(blur_u8_tile_kernel<CC, 5>);        \
        if (T.kxn == T.kyn && T.kxn == 7) return go(blur_u8_tile_kernel<CC, 7>);        \
        return go(blur_u8_tile_kernel<CC, 0>);                                          \
    }
    KB200_U8B(1) KB200_U8B(3) KB200_U8B(4)
#undef KB200_U8B
    return KB200_OK;
}

}  // namespace kb200

using namespace kb200;

extern "C" {

KB200_API void kb200_quantize_kernel_256(const float* kernel, uint32_t n, uint8_t* out) {
    if (kernel && out && n) quantize_kernel_256(kernel, (int)n, out);
}

KB200_API int kb200_gaussian_blur_u8(kb200_stream_t stream, const uint8_t* src, size_t src_len, uint8_t* dst, size_t dst_len, uint32_t cols,
                                     uint32_t rows, uint32_t channels, uint32_t batch, uint32_t ksize_x, uint32_t ksize_y, float sigma_x,
                                     float sigma_y) {
    uint32_t kxn, kyn;
    float sx, sy;
    KB200_TRY(kb200_gaussian_resolve(ksize_x, ksize_y, sigma_x, sigma_y, &kxn, &kyn, &sx, &sy));   // InvalidSigmaValue
    if (kxn > (uint32_t)U8B_MAXK || kyn > (uint32_t)U8B_MAXK)
        return fail(KB200_ERR_UNSUPPORTED, "gaussian_blur_u8 supports up to %d taps per axis, got (%u, %u)", U8B_MAXK, kxn, kyn);
    U8Taps T{};
    T.kxn = (int)kxn; T.kyn = (int)kyn;
    // blur_u8_path (filter/ops.rs:22-29)
    T.binomial = (kxn == 3 && kyn == 3 && sx >= 0.6f && sx <= 1.2f && sy >= 0.6f && sy <= 1.2f) ? 1 : 0;
    if (!T.binomial) {
        float fx[32], fy[32];
        kb200_gaussian_kernel_1d(kxn, sx, fx);
        kb200_gaussian_kernel_1d(kyn, sy, fy);
        quantize_kernel_256(fx, (int)kxn, T.kx);
        quantize_kernel_256(fy, (int)kyn, T.ky);
    }
    return launch_blur_u8(as_stream(stream), src, src_len, dst, dst_len, cols, rows, channels, batch, T);
}

KB200_API int kb200_box_blur_u8(kb200_stream_t stream, const uint8_t* src, size_t src_len, uint8_t* dst, size_t dst_len, uint32_t cols,
                                uint32_t rows, uint32_t channels, uint32_t batch, uint32_t ksize_x, uint32_t ksize_y) {
    if (ksize_x == 0 || ksize_y == 0 || ksize_x % 2 == 0 || ksize_y % 2 == 0)   // filter/ops.rs:74-76: InvalidSigmaValue(kx, ky)
        return fail(KB200_ERR_INVALID_KERNEL, "Invalid sigma value: (%g, %g)", (double)ksize_x, (double)ksize_y);
    if (ksize_x > (uint32_t)U8B_MAXK || ksize_y > (uint32_t)U8B_MAXK)
        return fail(KB200_ERR_UNSUPPORTED, "box_blur_u8 supports up to %d taps per axis, got (%u, %u)", U8B_MAXK, ksize_x, ksize_y);
    U8Taps T{};
    T.kxn = (int)ksize_x; T.kyn = (int)ksize_y; T.binomial = 0;
    float fx[32], fy[32];
    for (uint32_t i = 0; i < ksize_x; ++i) fx[i] = 1.0f / (float)ksize_x;   // filter/kernels.rs:10-13
    for (uint32_t i = 0; i < ksize_y; ++i) fy[i] = 1.0f / (float)ksize_y;
    quantize_kernel_256(fx, (int)ksize_x, T.kx);
    quantize_kernel_256(fy, (int)ksize_y, T.ky);
    return launch_blur_u8(as_stream(stream), src, src_len, dst, dst_len, cols, rows, channels, batch, T);
}

}  // extern "C"
