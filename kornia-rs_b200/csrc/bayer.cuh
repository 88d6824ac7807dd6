// bayer.cuh — bilinear demosaic of Bayer mosaics, 8-bit, 16-bit or MIPI-packed 10/12/14-bit samples, shared by the
// standalone decoders (color.cu: rgb_from_bayer_vec<T, P>, rgb_from_bayer_generic<T, P>) and the camera preprocess
// (preprocess.cu: preprocess_bayer_identity_kernel<OUT, T, P> and the Bayer taps of the generic kernel).  Everything
// here is generic over the sample type T; BayerSample<T> holds the few facts of T the kernels above it need.  Packed
// samples (T = BayerPacked<BITS>) only change the loads: they are unpacked into the words of the 16-bit kernels
// (bayer_unpack, bayer_load_rows_packed, bayer_px_packed), and everything after that is the uint16_t path.
//
// An extension beyond the reference, pinned to OpenCV: bit-identical to cv2.cvtColor(raw, COLOR_Bayer??2RGB)
// (checked against cv2 4.13 on 8-bit and 16-bit mosaics, tests/golden/bayer_cv2.npz and bayer16_cv2.npz).  A pattern (kb200_bayer_pattern) is named by its 2x2 quad
// read row-major: RGGB means the top-left pixel is R.  cv2's codes are offset from these names:
//     RGGB <-> COLOR_BayerBG2RGB, BGGR <-> COLOR_BayerRG2RGB, GRBG <-> COLOR_BayerGB2RGB, GBRG <-> COLOR_BayerGR2RGB.
//
// Output pixel (x, y) of a w x h frame p (w, h >= 3): cx = clamp(x, 1, w-2), cy = clamp(y, 1, h-2) — the border rows
// and columns copy their inner neighbour, corners included.  At (cx, cy), with N S W E the edge neighbours and D the
// sum of the four diagonal ones:
//     R or B site: own channel = p[cy][cx], G = (N+S+W+E+2) >> 2, the other of R / B = (D+2) >> 2;
//     G site:      G = p[cy][cx], the colour of the horizontal neighbours = (W+E+1) >> 1, of the vertical (N+S+1) >> 1.
#pragma once

#include "kb200_common.cuh"

namespace kb200 {

// Column / row parity of the R site in the quad of pattern P; the B site is at the opposite parities.
__host__ __device__ constexpr int bayer_rx(int P) { return (P == KB200_BAYER_BGGR || P == KB200_BAYER_GRBG) ? 1 : 0; }
__host__ __device__ constexpr int bayer_ry(int P) { return (P == KB200_BAYER_BGGR || P == KB200_BAYER_GBRG) ? 1 : 0; }

// The demosaiced colour of a centre pixel of column parity px, row parity py: c the centre sample, n s w e its edge
// neighbours, d the sum of its diagonal neighbours.  With P, px and py known at compile time this is two sums.
__device__ __forceinline__ void bayer_demosaic(int P, int px, int py, int c, int n, int s, int w, int e, int d, int& r, int& g, int& b) {
    const int rx = bayer_rx(P), ry = bayer_ry(P);
    if (px == rx && py == ry) {
        r = c; g = (n + s + w + e + 2) >> 2; b = (d + 2) >> 2;
    } else if (px != rx && py != ry) {
        b = c; g = (n + s + w + e + 2) >> 2; r = (d + 2) >> 2;
    } else {
        g = c;
        const int hz = (w + e + 1) >> 1, vt = (n + s + 1) >> 1;
        if (py == ry) { r = hz; b = vt; } else { r = vt; b = hz; }   // a G on an R row has R left and right
    }
}

// Output pixel (x, y) of a frame at `src` with row pitch `pitch` (in samples): nine sample loads around the clamped
// centre.  T = uint8_t (8-bit mosaics) or uint16_t (10- to 16-bit mosaics, one LSB-aligned word per sample): every sum
// is an int, so 4 * 65535 + 2 fits.
template <typename T>
__device__ __forceinline__ void bayer_px(const T* __restrict__ src, size_t pitch, int w, int h, int x, int y, int P, int rgb[3]) {
    const int cx = min(max(x, 1), w - 2), cy = min(max(y, 1), h - 2);
    const T* up = src + (size_t)(cy - 1) * pitch + cx;
    const T* mid = up + pitch;
    const T* dn = mid + pitch;
    const int d = (int)__ldg(up - 1) + (int)__ldg(up + 1) + (int)__ldg(dn - 1) + (int)__ldg(dn + 1);
    bayer_demosaic(P, cx & 1, cy & 1, __ldg(mid), __ldg(up), __ldg(dn), __ldg(mid - 1), __ldg(mid + 1), d, rgb[0], rgb[1], rgb[2]);
}

// MIPI CSI-2 packed samples of BITS = 10, 12 or 14 bits (V4L2's SRGGB10P ... SGBRG14P).  Each row is packed on its own
// in groups of G = 4, 2, 4 samples in GB = 5, 3, 7 bytes: the first G bytes hold the high 8 bits of each sample, the
// rest the low BITS - 8 bits of sample j at bit (BITS - 8) * j of their little-endian word.  A tag type: no value of it
// is ever read, it only selects the packed loaders below.
template <int BITS> struct BayerPacked {};
__host__ __device__ constexpr int bayer_packed_group(int bits) { return bits == 12 ? 2 : 4; }
__host__ __device__ constexpr int bayer_packed_group_bytes(int bits) { return bayer_packed_group(bits) * bits / 8; }

// The sample types: uint8_t (8-bit mosaics), uint16_t (10- to 16-bit) and BayerPacked<BITS>.  VEC_COLS: columns per
// decoder thread (one 16-byte vector of uint8_t / uint16_t samples).  ID_WORDS: 32-bit words per 4-sample load of the
// preprocess identity kernel (LDG.32 / LDG.64), and ID_ALIGN: the row and frame alignment in bytes that load needs.
// Word: the sample type of the unpacked words the demosaic reads (bayer_row) and of the decoder's output.  PACKED_BITS:
// the packing's bits per sample, 0 for the unpacked types.
template <typename T> struct BayerSample;
template <> struct BayerSample<uint8_t> {
    static constexpr uint32_t VEC_COLS = 16, ID_WORDS = 1, ID_ALIGN = 4;
    static constexpr int PACKED_BITS = 0;
    using Word = uint8_t;
};
template <> struct BayerSample<uint16_t> {
    static constexpr uint32_t VEC_COLS = 8, ID_WORDS = 2, ID_ALIGN = 8;
    static constexpr int PACKED_BITS = 0;
    using Word = uint16_t;
};
template <int BITS> struct BayerSample<BayerPacked<BITS>> {
    static constexpr uint32_t VEC_COLS = 8, ID_WORDS = 2, ID_ALIGN = 16;
    static constexpr int PACKED_BITS = BITS;
    using Word = uint16_t;
};

// Sample x of a packed row at `row` (bits known at compile time in the fast kernels, at run time in the generic
// preprocess): the high byte and the low field of its group, reading no byte outside the group.
// Shifts, not divisions: with bits known only at run time a division by the group size is a long integer sequence.
__device__ __forceinline__ int bayer_packed_sample(const uint8_t* __restrict__ row, int x, int bits) {
    const int gs = bits == 12 ? 1 : 2, lo = bits - 8;   // log2 of the samples per group, low bits per sample
    const int j = x & ((1 << gs) - 1);
    const uint8_t* grp = row + (x >> gs) * ((bits << gs) >> 3);
    const int at = lo * j, bi = at >> 3, sh = at & 7;
    int field = __ldg(grp + (1 << gs) + bi);
    if (sh + lo > 8) field |= (int)__ldg(grp + (1 << gs) + bi + 1) << 8;
    return ((int)__ldg(grp + j) << lo) | ((field >> sh) & ((1 << lo) - 1));
}

// bayer_px on a packed frame: `pitch` in bytes.
__device__ __forceinline__ void bayer_px_packed(const uint8_t* __restrict__ src, size_t pitch, int w, int h, int x, int y, int P, int bits,
                                                int rgb[3]) {
    const int cx = min(max(x, 1), w - 2), cy = min(max(y, 1), h - 2);
    const uint8_t* up = src + (size_t)(cy - 1) * pitch;
    const uint8_t* mid = up + pitch;
    const uint8_t* dn = mid + pitch;
    auto at = [&](const uint8_t* row, int c) { return bayer_packed_sample(row, c, bits); };
    const int d = at(up, cx - 1) + at(up, cx + 1) + at(dn, cx - 1) + at(dn, cx + 1);
    bayer_demosaic(P, cx & 1, cy & 1, at(mid, cx), at(up, cx), at(dn, cx), at(mid, cx - 1), at(mid, cx + 1), d, rgb[0], rgb[1], rgb[2]);
}

// Unpacks the N samples of whole groups held in `bytes` (little-endian, byte 0 the first byte of a group) into N / 2
// words of 16-bit samples, sample 2m in the low half of word m: the layout bayer_row reads for uint16_t.
template <int BITS, int N>
__device__ __forceinline__ void bayer_unpack(const uint32_t* bytes, uint32_t words[N / 2]) {
    constexpr int G = bayer_packed_group(BITS), GB = bayer_packed_group_bytes(BITS), LO = BITS - 8;
    auto byte = [&](int k) { return (bytes[k >> 2] >> (8 * (k & 3))) & 0xFFu; };
#pragma unroll
    for (int s = 0; s < N; ++s) {
        const int base = (s / G) * GB, j = s % G, at = LO * j;
        uint32_t field = byte(base + G + (at >> 3));
        if ((at & 7) + LO > 8) field |= byte(base + G + (at >> 3) + 1) << 8;
        const uint32_t v = (byte(base + j) << LO) | ((field >> (at & 7)) & ((1u << LO) - 1u));
        if (s & 1) words[s >> 1] |= v << 16; else words[s >> 1] = v;
    }
}

// Samples of type T per 32-bit word of a row segment, and their width in bits.
template <typename T> __host__ __device__ constexpr int bayer_per_word() { return 4 / (int)sizeof(T); }
template <typename T> __host__ __device__ constexpr int bayer_bits() { return 8 * (int)sizeof(T); }

// Sample j of a row segment of NW words, j = -1 and j = S*NW (S samples per word) being the halo samples left and
// right of it.
template <int NW, typename T = uint8_t>
__device__ __forceinline__ int bayer_seg_sample(const uint32_t w[NW], int left, int right, int j) {
    constexpr int S = bayer_per_word<T>(), B = bayer_bits<T>();
    constexpr uint32_t M = (1u << B) - 1u;
    return j < 0 ? left : j >= S * NW ? right : (int)((w[j / S] >> (B * (j % S))) & M);
}

// The S*NW demosaiced pixels of one row segment of the fast kernels: row parity PY, the segment starting at an even
// column.  n / c / s: the segments of the rows above, at and below; hl / hr: their halo samples (above, at, below).
// left_edge / right_edge: the segment holds column 0 / w-1, which copy columns 1 / w-2.
template <int P, int PY, int NW, typename T = uint8_t>
__device__ __forceinline__ void bayer_row(const uint32_t n[NW], const uint32_t c[NW], const uint32_t s[NW], const int hl[3], const int hr[3],
                                          bool left_edge, bool right_edge, int r[bayer_per_word<T>() * NW],
                                          int g[bayer_per_word<T>() * NW], int b[bayer_per_word<T>() * NW]) {
    constexpr int N = bayer_per_word<T>() * NW;
#pragma unroll
    for (int j = 0; j < N; ++j) {
        const int d = bayer_seg_sample<NW, T>(n, hl[0], hr[0], j - 1) + bayer_seg_sample<NW, T>(n, hl[0], hr[0], j + 1) +
                      bayer_seg_sample<NW, T>(s, hl[2], hr[2], j - 1) + bayer_seg_sample<NW, T>(s, hl[2], hr[2], j + 1);
        bayer_demosaic(P, j & 1, PY, bayer_seg_sample<NW, T>(c, hl[1], hr[1], j), bayer_seg_sample<NW, T>(n, hl[0], hr[0], j),
                       bayer_seg_sample<NW, T>(s, hl[2], hr[2], j), bayer_seg_sample<NW, T>(c, hl[1], hr[1], j - 1),
                       bayer_seg_sample<NW, T>(c, hl[1], hr[1], j + 1), d, r[j], g[j], b[j]);
    }
    constexpr int L = N - 1;
    if (left_edge) { r[0] = r[1]; g[0] = g[1]; b[0] = b[1]; }
    if (right_edge) { r[L] = r[L - 1]; g[L] = g[L - 1]; b[L] = b[L - 1]; }
}

// Loads the four rows ya-1 .. ya+2 of a lane's NW-word segment at column x (row index clamped to h-1: row ya+2 = h
// when h is odd is never used), and the halo sample on each side of it.  `pitch` is in samples.  The halos come from
// the neighbouring lanes' words by shuffle; the warp's edge lanes load theirs.  Every lane of the warp must call; a lane
// whose neighbour holds another row pair's segment has its halo there at column -1 or w, which the border copy never reads.
template <int NW, typename T, typename LOAD>
__device__ __forceinline__ void bayer_load_rows(const T* __restrict__ frame, size_t pitch, uint32_t w, uint32_t h, uint32_t x,
                                                uint32_t ya, uint32_t lane, LOAD load, uint32_t rows[4][NW], int hl[4], int hr[4]) {
    constexpr int S = bayer_per_word<T>(), B = bayer_bits<T>();
    constexpr uint32_t M = (1u << B) - 1u;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const T* row = frame + (size_t)min(ya - 1 + k, h - 1) * pitch;
        load(row + x, rows[k]);
        hl[k] = (int)(__shfl_up_sync(0xFFFFFFFFu, rows[k][NW - 1], 1) >> (32 - B));
        hr[k] = (int)(__shfl_down_sync(0xFFFFFFFFu, rows[k][0], 1) & M);
        if (lane == 0 && x > 0) hl[k] = __ldg(row + x - 1);
        if (lane == 31 && x + S * NW < w) hr[k] = __ldg(row + x + S * NW);
    }
}

// bayer_load_rows on a packed frame of BITS-bit samples (`pitch` in bytes): LOAD(k, row, words) fills the NW words of
// the lane's 2 * NW columns at x of row ya-1+k (clamped) in the uint16_t layout (bayer_unpack), and the edge lanes read
// their halo sample from its group.
template <int NW, int BITS, typename LOAD>
__device__ __forceinline__ void bayer_load_rows_packed(const uint8_t* __restrict__ frame, size_t pitch, uint32_t w, uint32_t h, uint32_t x,
                                                       uint32_t ya, uint32_t lane, LOAD load, uint32_t rows[4][NW], int hl[4], int hr[4]) {
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const uint8_t* row = frame + (size_t)min(ya - 1 + k, h - 1) * pitch;
        load(k, row, rows[k]);
        hl[k] = (int)(__shfl_up_sync(0xFFFFFFFFu, rows[k][NW - 1], 1) >> 16);
        hr[k] = (int)(__shfl_down_sync(0xFFFFFFFFu, rows[k][0], 1) & 0xFFFFu);
        if (lane == 0 && x > 0) hl[k] = bayer_packed_sample(row, (int)x - 1, BITS);
        if (lane == 31 && x + 2 * NW < w) hr[k] = bayer_packed_sample(row, (int)(x + 2 * NW), BITS);
    }
}

// Number of row pairs the fast kernels walk: rows (1 + 2k, 2 + 2k) cover the interior rows 1 .. h-2 (the second row
// of the last pair is h-1, a copy of h-2, when h is odd); the thread of pair 0 also writes row 0 and the thread whose
// second row is h-2 also writes row h-1.
__host__ __device__ inline uint32_t bayer_row_pairs(uint32_t h) { return (h - 1) / 2; }

}  // namespace kb200
