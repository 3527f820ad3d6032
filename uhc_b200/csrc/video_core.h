// video_core.h -- the per-block arithmetic of the baseline JPEG encoder (ITU-T T.81), shared by the kernels (video.cu) and the host emulation
// (tests/emu/video_emu.cpp, -DUHC_EMU).  Integer arithmetic only, so the device's bytes equal the emulation's bytes.
//
// One fixed format: JFIF, full-range BT.601 YCbCr, 4:2:0 (a 16 x 16 MCU = Y0 Y1 Y2 Y3 Cb Cr), the Annex K quantisation tables scaled as IJG does
// and the four Annex K Huffman tables, restart interval = one MCU row.
//   colour     Y  = (19595 R + 38470 G +  7471 B + 32768) >> 16
//              Cb = (-11059 R - 21709 G + 32768 B + (128 << 16) + 32767) >> 16, Cr = (32768 R - 27439 G - 5329 B + (128 << 16) + 32767) >> 16
//              (16-bit constants, each row summing to 65536 or 0; every sum is >= 0 before the shift, so the shift is a floor; the chroma rounding
//              term is one below a half, as IJG's, so that pure blue / red give Cb / Cr = 255, not 256: every sample is in 0 .. 255); a chroma sample is
//              the mean of its 2 x 2 full-resolution values, (sum + 2) >> 2.  Pixels past the right / bottom edge repeat the last column / row.
//   DCT        s = sample - 128; rows t[y][u] = (sum_x K[u][x] s[y][x] + 256) >> 9 with K = round(8192 alpha(u) cos((2x + 1) u pi / 16)) (13-bit
//              constants, |t| < 2^13: 4 fractional bits), then columns X[v][u] = sum_y K[v][y] t[y][u] (|X| < 2^28, int32): X = 2^17 F where F is
//              the orthonormal DCT-II (JPEG's FDCT) up to the constants' and the row shift's rounding.
//   quantise   q = sign(X) ((|X| + Q 2^16) / (Q 2^17)): |F| / Q rounded half away from zero in one integer division; AC clamped to +-1023, DC to
//              +-1023, so every DC difference is within the +-2047 baseline codes.
#pragma once
#include <stdint.h>
#include <stddef.h>

#if defined(UHC_EMU)
#define UHC_VHD inline
#else
#define UHC_VHD __host__ __device__ inline
#endif

namespace uhc {
namespace jpeg {

constexpr int MAX_WH = 16384;
constexpr int BLK = 6;                        // blocks per MCU
// worst-case bits of one block: DC code (<= 11) + 11 magnitude bits, 63 AC codes (<= 16) + 10 magnitude bits, the EOB (<= 16)
constexpr int BLOCK_BITS_MAX = 11 + 11 + 63 * (16 + 10) + 16;
// fixed-size parts of a frame: SOI, APP0 (18), DQT x 2 (69), SOF0 (19), DHT (33, 33, 183, 183), DRI (6), SOS (14); and EOI
constexpr int HEADER_BYTES = 2 + 18 + 2 * 69 + 19 + 33 + 33 + 183 + 183 + 6 + 14;

struct Tables {
    uint16_t code[4][256];                    // [DC lum, AC lum, DC chroma, AC chroma][symbol] canonical Huffman code
    uint8_t size[4][256];                     // its length in bits (0: not in the table)
};

struct Quant {
    int q[2][64];                             // [lum, chroma][natural order] 1 .. 255
    uint8_t zigzag[64];                       // natural index of zigzag position k (a copy of ZIGZAG the kernels read from their parameters)
};

static const uint8_t ZIGZAG[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                                   41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                                   30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

// ---- host only: the Annex K tables, the header and the quality scaling
static const uint8_t QLUM[64] = {16, 11, 10, 16, 24,  40,  51,  61,  12, 12, 14, 19, 26,  58,  60,  55,  14, 13, 16, 24, 40,  57,
                                 69, 56, 14, 17, 22,  29,  51,  87,  80, 62, 18, 22, 37,  56,  68,  109, 103, 77, 24, 35, 55, 64,
                                 81, 104, 113, 92, 49, 64, 78,  87,  103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99};
static const uint8_t QCHR[64] = {17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99, 24, 26, 56, 99, 99, 99,
                                 99, 99, 47, 66, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99,
                                 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99};
static const uint8_t BITS_DCL[16] = {0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0};
static const uint8_t BITS_DCC[16] = {0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0};
static const uint8_t VALS_DC[12] = {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11};
static const uint8_t BITS_ACL[16] = {0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7d};
static const uint8_t VALS_ACL[162] = {
    0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07, 0x22, 0x71, 0x14, 0x32, 0x81, 0x91, 0xa1,
    0x08, 0x23, 0x42, 0xb1, 0xc1, 0x15, 0x52, 0xd1, 0xf0, 0x24, 0x33, 0x62, 0x72, 0x82, 0x09, 0x0a, 0x16, 0x17, 0x18, 0x19, 0x1a, 0x25, 0x26,
    0x27, 0x28, 0x29, 0x2a, 0x34, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56,
    0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x83, 0x84, 0x85,
    0x86, 0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9, 0xaa,
    0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6,
    0xd7, 0xd8, 0xd9, 0xda, 0xe1, 0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf1, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9,
    0xfa};
static const uint8_t BITS_ACC[16] = {0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77};
static const uint8_t VALS_ACC[162] = {
    0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61, 0x71, 0x13, 0x22, 0x32, 0x81, 0x08, 0x14, 0x42,
    0x91, 0xa1, 0xb1, 0xc1, 0x09, 0x23, 0x33, 0x52, 0xf0, 0x15, 0x62, 0x72, 0xd1, 0x0a, 0x16, 0x24, 0x34, 0xe1, 0x25, 0xf1, 0x17, 0x18, 0x19,
    0x1a, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55,
    0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x82, 0x83,
    0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8,
    0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4,
    0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9,
    0xfa};

// canonical codes (T.81 Annex C) of the four tables
inline void make_tables(Tables &t) {
    const uint8_t *bits[4] = {BITS_DCL, BITS_ACL, BITS_DCC, BITS_ACC};
    const uint8_t *vals[4] = {VALS_DC, VALS_ACL, VALS_DC, VALS_ACC};
    for (int k = 0; k < 4; k++) {
        for (int s = 0; s < 256; s++) { t.code[k][s] = 0; t.size[k][s] = 0; }
        unsigned code = 0;
        int i = 0;
        for (int len = 1; len <= 16; len++, code <<= 1)
            for (int j = 0; j < bits[k][len - 1]; j++, i++, code++) { t.code[k][vals[k][i]] = (uint16_t)code; t.size[k][vals[k][i]] = (uint8_t)len; }
    }
}

// IJG's scaling of the Annex K tables: scale = q < 50 ? 5000 / q : 200 - 2q, entry = (base * scale + 50) / 100 clamped to 1 .. 255
inline void make_quant(int quality, Quant &qt) {
    const int scale = quality < 50 ? 5000 / quality : 200 - 2 * quality;
    for (int i = 0; i < 64; i++) {
        const int a = (QLUM[i] * scale + 50) / 100, b = (QCHR[i] * scale + 50) / 100;
        qt.q[0][i] = a < 1 ? 1 : a > 255 ? 255 : a;
        qt.q[1][i] = b < 1 ? 1 : b > 255 ? 255 : b;
        qt.zigzag[i] = ZIGZAG[i];
    }
}

// the HEADER_BYTES bytes before the first entropy-coded segment
inline void make_header(int W, int H, const Quant &qt, uint8_t *h) {
    int k = 0;
    auto b = [&](int v) { h[k++] = (uint8_t)v; };
    auto w = [&](int v) { b(v >> 8); b(v & 255); };
    w(0xFFD8);
    w(0xFFE0); w(16); b('J'); b('F'); b('I'); b('F'); b(0); b(1); b(1); b(0); w(1); w(1); b(0); b(0);
    for (int c = 0; c < 2; c++) { w(0xFFDB); w(67); b(c); for (int i = 0; i < 64; i++) b(qt.q[c][ZIGZAG[i]]); }
    w(0xFFC0); w(17); b(8); w(H); w(W); b(3);
    b(1); b(0x22); b(0); b(2); b(0x11); b(1); b(3); b(0x11); b(1);
    const uint8_t *bits[4] = {BITS_DCL, BITS_ACL, BITS_DCC, BITS_ACC};
    const uint8_t *vals[4] = {VALS_DC, VALS_ACL, VALS_DC, VALS_ACC};
    const int cls[4] = {0x00, 0x10, 0x01, 0x11};
    for (int t = 0; t < 4; t++) {
        int nv = 0;
        for (int i = 0; i < 16; i++) nv += bits[t][i];
        w(0xFFC4); w(3 + 16 + nv); b(cls[t]);
        for (int i = 0; i < 16; i++) b(bits[t][i]);
        for (int i = 0; i < nv; i++) b(vals[t][i]);
    }
    w(0xFFDD); w(4); w((W + 15) / 16);
    w(0xFFDA); w(12); b(3); b(1); b(0x00); b(2); b(0x11); b(3); b(0x11); b(0); b(63); b(0);
}

// MCU grid of a frame
UHC_VHD int mcu_cols(int W) { return (W + 15) / 16; }
UHC_VHD int mcu_rows(int H) { return (H + 15) / 16; }

// the worst case of one frame: every block at BLOCK_BITS_MAX plus a byte of padding per segment, every byte stuffed, the RST markers, the
// headers and EOI.  A true bound for any input: the block bound holds for any coefficients the quantiser can produce.
UHC_VHD size_t frame_bound(int W, int H) {
    const size_t seg = ((size_t)mcu_cols(W) * BLK * BLOCK_BITS_MAX + 7) / 8 + 1;
    return (size_t)HEADER_BYTES + (size_t)mcu_rows(H) * (2 * seg + 2) + 2;
}

// the level-shifted samples [6][64] (natural order) of MCU (mx, my) of one frame rgb [H][W][3]
UHC_VHD void mcu_samples(const uint8_t *rgb, int W, int H, int mx, int my, int comp_block, int *s) {
    if (comp_block < 4) {
        const int x0 = mx * 16 + (comp_block & 1) * 8, y0 = my * 16 + (comp_block >> 1) * 8;
        for (int y = 0; y < 8; y++)
            for (int x = 0; x < 8; x++) {
                const int px = x0 + x < W ? x0 + x : W - 1, py = y0 + y < H ? y0 + y : H - 1;
                const uint8_t *p = rgb + ((size_t)py * W + px) * 3;
                s[y * 8 + x] = ((19595 * p[0] + 38470 * p[1] + 7471 * p[2] + 32768) >> 16) - 128;
            }
        return;
    }
    const bool cb = comp_block == 4;
    for (int y = 0; y < 8; y++)
        for (int x = 0; x < 8; x++) {
            int sum = 0;
            for (int j = 0; j < 4; j++) {
                const int xx = mx * 16 + 2 * x + (j & 1), yy = my * 16 + 2 * y + (j >> 1);
                const int px = xx < W ? xx : W - 1, py = yy < H ? yy : H - 1;
                const uint8_t *p = rgb + ((size_t)py * W + px) * 3;
                const int r = p[0], g = p[1], b = p[2];
                sum += cb ? (-11059 * r - 21709 * g + 32768 * b + (128 << 16) + 32767) >> 16
                          : (32768 * r - 27439 * g - 5329 * b + (128 << 16) + 32767) >> 16;
            }
            s[y * 8 + x] = ((sum + 2) >> 2) - 128;
        }
}

// X = 2^17 F (natural order) of level-shifted samples s[64]
UHC_VHD void fdct(const int *s, int *X) {
    const int K[8][8] = {{2896, 2896, 2896, 2896, 2896, 2896, 2896, 2896},    {4017, 3406, 2276, 799, -799, -2276, -3406, -4017},
                         {3784, 1567, -1567, -3784, -3784, -1567, 1567, 3784}, {3406, -799, -4017, -2276, 2276, 4017, 799, -3406},
                         {2896, -2896, -2896, 2896, 2896, -2896, -2896, 2896}, {2276, -4017, 799, 3406, -3406, -799, 4017, -2276},
                         {1567, -3784, 3784, -1567, -1567, 3784, -3784, 1567}, {799, -2276, 3406, -4017, 4017, -3406, 2276, -799}};
    int t[64];
    for (int y = 0; y < 8; y++)
        for (int u = 0; u < 8; u++) {
            int a = 0;
            for (int x = 0; x < 8; x++) a += K[u][x] * s[y * 8 + x];
            t[y * 8 + u] = (a + 256) >> 9;
        }
    for (int v = 0; v < 8; v++)
        for (int u = 0; u < 8; u++) {
            int a = 0;
            for (int y = 0; y < 8; y++) a += K[v][y] * t[y * 8 + u];
            X[v * 8 + u] = a;
        }
}

// X (natural order) -> quantised coefficients in zigzag order
UHC_VHD void quantise(const int *X, const Quant &qt, int comp, int16_t *zz) {
    for (int k = 0; k < 64; k++) {
        const int i = qt.zigzag[k], Q = qt.q[comp][i], a = X[i] < 0 ? -X[i] : X[i];
        int v = (a + (Q << 16)) / (Q << 17);
        v = v > 1023 ? 1023 : v;
        zz[k] = (int16_t)(X[i] < 0 ? -v : v);
    }
}

// block b (0..3 Y, 4 Cb, 5 Cr) of MCU (mx, my): samples, DCT, quantisation
UHC_VHD void encode_block(const uint8_t *rgb, int W, int H, int mx, int my, int b, const Quant &qt, int16_t *zz) {
    int s[64], X[64];
    mcu_samples(rgb, W, H, mx, my, b, s);
    fdct(s, X);
    quantise(X, qt, b < 4 ? 0 : 1, zz);
}

UHC_VHD int magnitude_bits(int v) {
    int a = v < 0 ? -v : v, n = 0;
    while (a) { n++; a >>= 1; }
    return n;
}

// the Huffman coding of one block, as (bits, length) pairs of at most 27 bits to put(): DC difference against pred, then the AC run lengths
// (ZRL for 16 zeros, EOB after the last non-zero coefficient).  table: 0 for Y, 2 for chroma (the AC table is table + 1).
template <class Put>
UHC_VHD void code_block(const int16_t *zz, int pred, const Tables &t, int table, Put &put) {
    const int d = zz[0] - pred, nd = magnitude_bits(d);
    put(((unsigned)t.code[table][nd] << nd) | ((unsigned)(d < 0 ? d - 1 : d) & ((1u << nd) - 1)), t.size[table][nd] + nd);
    const int ac = table + 1;
    int run = 0;
    for (int k = 1; k < 64; k++) {
        const int v = zz[k];
        if (v == 0) { run++; continue; }
        for (; run >= 16; run -= 16) put(t.code[ac][0xF0], t.size[ac][0xF0]);
        const int n = magnitude_bits(v), sym = (run << 4) | n;
        put(((unsigned)t.code[ac][sym] << n) | ((unsigned)(v < 0 ? v - 1 : v) & ((1u << n) - 1)), t.size[ac][sym] + n);
        run = 0;
    }
    if (run) put(t.code[ac][0], t.size[ac][0]);
}

struct CountBits {
    int n = 0;
    UHC_VHD void operator()(unsigned, int len) { n += len; }
};

// the DC predictor of block b of MCU column mx in its segment (one MCU row): the previous block of the same component, 0 at the row's start
UHC_VHD int prev_block(int mx, int b) {
    if (b >= 1 && b <= 3) return mx * BLK + b - 1;
    if (mx == 0) return -1;
    return (mx - 1) * BLK + (b == 0 ? 3 : b);
}

}  // namespace jpeg
}  // namespace uhc
