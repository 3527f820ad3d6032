// video_emu.cpp -- TEST INFRASTRUCTURE: the JPEG encoder's per-block arithmetic (uhc_b200/csrc/video_core.h) compiled as host code (-DUHC_EMU)
// around a serial bit writer, so the kernels' coefficients are checked against an fp64 DCT on a CPU-only box and the GPU's bytes against these
// byte for byte.  Never loaded by the product path (uhc_b200/engine.py only loads the CUDA library).
#define UHC_EMU 1
#include <stdint.h>
#include <string.h>
#include <vector>
#include "../../uhc_b200/csrc/video_core.h"

using namespace uhc;

namespace {

struct SerialBits {
    std::vector<uint8_t> *out;
    uint64_t acc = 0;
    int nacc = 0;
    void byte(unsigned v) { out->push_back((uint8_t)v); if (v == 0xFF) out->push_back(0); }
    void operator()(unsigned v, int len) {
        acc = (acc << len) | v; nacc += len;
        while (nacc >= 8) { nacc -= 8; byte((unsigned)(acc >> nacc) & 255u); }
    }
    void flush() { if (nacc) (*this)((1u << (8 - nacc)) - 1, 8 - nacc); }   // 1-bits to the byte boundary
};

void frame_coefs(const uint8_t *rgb, int W, int H, const jpeg::Quant &qt, int16_t *coef) {
    const int mx = jpeg::mcu_cols(W), my = jpeg::mcu_rows(H);
    for (int y = 0; y < my; y++)
        for (int x = 0; x < mx; x++)
            for (int b = 0; b < jpeg::BLK; b++) jpeg::encode_block(rgb, W, H, x, y, b, qt, coef + (((size_t)y * mx + x) * jpeg::BLK + b) * 64);
}

}  // namespace

extern "C" {

size_t emu_jpeg_bound(int W, int H) { return jpeg::frame_bound(W, H); }

// X = 2^17 F of n level-shifted blocks s [n][64] (natural order)
void emu_jpeg_fdct(long n, const int *s, int *X) {
    for (long i = 0; i < n; i++) jpeg::fdct(s + 64 * i, X + 64 * i);
}

// the quantisation table [2][64] (natural order) of a quality
void emu_jpeg_quant(int quality, int *q) {
    jpeg::Quant qt;
    jpeg::make_quant(quality, qt);
    memcpy(q, qt.q, sizeof(qt.q));
}

// quantised coefficients [n][mcu rows][mcu cols][6][64] (zigzag) of n frames rgb [n][H][W][3]
void emu_jpeg_coefs(const uint8_t *rgb, long n, int W, int H, int quality, int16_t *coef) {
    jpeg::Quant qt;
    jpeg::make_quant(quality, qt);
    const size_t per = (size_t)jpeg::mcu_cols(W) * jpeg::mcu_rows(H) * jpeg::BLK * 64;
    for (long f = 0; f < n; f++) frame_coefs(rgb + (size_t)f * H * W * 3, W, H, qt, coef + f * per);
}

// uhc_jpeg_encode on the host, one block after the other: returns the total bytes; writes out (and offsets [n + 1]) when total <= cap
size_t emu_jpeg_encode(const uint8_t *rgb, long n, int W, int H, int quality, uint8_t *out, size_t cap, size_t *offsets) {
    jpeg::Quant qt;
    jpeg::make_quant(quality, qt);
    jpeg::Tables tab;
    jpeg::make_tables(tab);
    const int mx = jpeg::mcu_cols(W), my = jpeg::mcu_rows(H);
    std::vector<int16_t> coef((size_t)mx * my * jpeg::BLK * 64);
    std::vector<uint8_t> all;
    std::vector<size_t> offs(1, 0);
    for (long f = 0; f < n; f++) {
        frame_coefs(rgb + (size_t)f * H * W * 3, W, H, qt, coef.data());
        std::vector<uint8_t> file(jpeg::HEADER_BYTES);
        jpeg::make_header(W, H, qt, file.data());
        for (int y = 0; y < my; y++) {
            if (y > 0) { file.push_back(0xFF); file.push_back((uint8_t)(0xD0 + ((y - 1) & 7))); }
            SerialBits bw;
            bw.out = &file;
            const int16_t *row = coef.data() + (size_t)y * mx * jpeg::BLK * 64;
            for (int x = 0; x < mx; x++)
                for (int b = 0; b < jpeg::BLK; b++) {
                    const int p = jpeg::prev_block(x, b);
                    jpeg::code_block(row + ((size_t)x * jpeg::BLK + b) * 64, p < 0 ? 0 : row[(size_t)p * 64], tab, b < 4 ? 0 : 2, bw);
                }
            bw.flush();
        }
        file.push_back(0xFF); file.push_back(0xD9);
        all.insert(all.end(), file.begin(), file.end());
        offs.push_back(all.size());
    }
    if (all.size() <= cap) {
        if (!all.empty()) memcpy(out, all.data(), all.size());
        if (offsets) memcpy(offsets, offs.data(), offs.size() * sizeof(size_t));
    }
    return all.size();
}
}
