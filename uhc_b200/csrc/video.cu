// video.cu -- the batched baseline JPEG encoder behind the C ABI (include/uhc_video.h).  Frames are encoded in passes of at most SCRATCH_CAP
// bytes of scratch (at least one frame); per pass:
//   k_jpeg_blocks  one thread per 8 x 8 block, blockIdx.y = frame: colour, 4:2:0 mean, DCT, quantisation, zigzag (video_core.h) -> coef
//   k_jpeg_rows    one warp per entropy-coded segment (an MCU row): per block its bit count with the in-segment DC differences, a warp scan, the
//                  bits OR-ed into the segment's words (disjoint, so the merge is deterministic), 1-bit padding, the count of 0xFF bytes
//   k_jpeg_frame   one thread per frame: the segments' offsets behind the header and the RST markers, the frame's bytes
//   k_jpeg_write   one warp per segment: the header (segment 0), the RST marker before it, its bytes with a 0x00 after every 0xFF, EOI (last)
// The frame sizes come to the host between k_jpeg_frame and k_jpeg_write, which is where the frame offsets are scanned.  Every frame is
// encoded once: a call of several passes whose out_cap could be too small writes its files into a staging buffer (at most out_cap bytes, grown
// as the files arrive) and copies them to out_dev when the total is known to fit, so that -3 leaves out_dev untouched.
#include <cuda_runtime.h>
#include <string>
#include <vector>
#include "../../include/uhc_video.h"
#include "engine_slots.h"
#include "errors.h"
#include "video_core.h"

using namespace uhc;

namespace {

constexpr size_t SCRATCH_CAP = 256u << 20;   // coefficients + segment words of one pass
constexpr int ROW_WARPS = 4;

__constant__ jpeg::Tables c_tab;

struct Geometry {
    int W, H, mcux, mcuy, seg_words;
    long mcus;
};

Geometry geometry(int W, int H) {
    Geometry g;
    g.W = W; g.H = H; g.mcux = jpeg::mcu_cols(W); g.mcuy = jpeg::mcu_rows(H); g.mcus = (long)g.mcux * g.mcuy;
    g.seg_words = (int)(((size_t)g.mcux * jpeg::BLK * jpeg::BLOCK_BITS_MAX + 31) / 32 + 1);
    return g;
}

size_t frame_scratch(const Geometry &g) {
    return (size_t)g.mcus * jpeg::BLK * 64 * sizeof(int16_t) + (size_t)g.mcuy * g.seg_words * sizeof(uint32_t);
}

struct VideoCtx {
    int16_t *d_coef = nullptr; size_t coef_cap = 0;
    uint32_t *d_words = nullptr; size_t words_cap = 0;
    int *d_seg_raw = nullptr, *d_seg_len = nullptr; size_t *d_seg_off = nullptr; size_t seg_cap = 0;
    size_t *d_fsize = nullptr, *d_foff = nullptr, *h_fsize = nullptr; size_t frame_cap = 0;
    uint8_t *d_hdr = nullptr;
    unsigned char *d_stage = nullptr; size_t stage_cap = 0;         // the files of a multi-pass call that could overflow out_cap
};

VideoCtx *get_ctx(UhcEngine *e) {
    void *&s = engine_slot(e, SLOT_VIDEO);
    if (!s) s = new VideoCtx();
    return (VideoCtx *)s;
}

// grows every scratch array to hold nf frames of geometry g; the stream is synchronised first (an earlier call may still use the old arrays)
int reserve(VideoCtx *c, const Geometry &g, long nf, cudaStream_t st) {
    const size_t coef = (size_t)nf * g.mcus * jpeg::BLK * 64, words = (size_t)nf * g.mcuy * g.seg_words, seg = (size_t)nf * g.mcuy;
    if (coef <= c->coef_cap && words <= c->words_cap && seg <= c->seg_cap && (size_t)nf <= c->frame_cap && c->d_hdr) return 0;
    CK(cudaStreamSynchronize(st));
    if (coef > c->coef_cap) {
        cudaFree(c->d_coef); c->d_coef = nullptr; c->coef_cap = 0;
        CK(cudaMalloc((void **)&c->d_coef, coef * sizeof(int16_t))); c->coef_cap = coef;
    }
    if (words > c->words_cap) {
        cudaFree(c->d_words); c->d_words = nullptr; c->words_cap = 0;
        CK(cudaMalloc((void **)&c->d_words, words * sizeof(uint32_t))); c->words_cap = words;
    }
    if (seg > c->seg_cap) {
        cudaFree(c->d_seg_raw); cudaFree(c->d_seg_len); cudaFree(c->d_seg_off);
        c->d_seg_raw = c->d_seg_len = nullptr; c->d_seg_off = nullptr; c->seg_cap = 0;
        CK(cudaMalloc((void **)&c->d_seg_raw, seg * sizeof(int)));
        CK(cudaMalloc((void **)&c->d_seg_len, seg * sizeof(int)));
        CK(cudaMalloc((void **)&c->d_seg_off, seg * sizeof(size_t)));
        c->seg_cap = seg;
    }
    if ((size_t)nf > c->frame_cap) {
        cudaFree(c->d_fsize); cudaFree(c->d_foff); cudaFreeHost(c->h_fsize);
        c->d_fsize = c->d_foff = c->h_fsize = nullptr; c->frame_cap = 0;
        CK(cudaMalloc((void **)&c->d_fsize, nf * sizeof(size_t)));
        CK(cudaMalloc((void **)&c->d_foff, nf * sizeof(size_t)));
        CK(cudaMallocHost((void **)&c->h_fsize, nf * sizeof(size_t)));
        c->frame_cap = (size_t)nf;
    }
    if (!c->d_hdr) CK(cudaMalloc((void **)&c->d_hdr, jpeg::HEADER_BYTES));
    return 0;
}

// grows the staging buffer to hold `need` bytes (at most `limit`), keeping its first `keep` bytes
int reserve_stage(VideoCtx *c, size_t need, size_t keep, size_t limit, cudaStream_t st) {
    if (need <= c->stage_cap) return 0;
    size_t cap = c->stage_cap * 2 > need ? c->stage_cap * 2 : need;
    cap = cap < limit ? cap : limit;
    unsigned char *p = nullptr;
    CK(cudaMalloc((void **)&p, cap));
    if (keep) CK(cudaMemcpyAsync(p, c->d_stage, keep, cudaMemcpyDeviceToDevice, st));
    CK(cudaStreamSynchronize(st));                                  // the old buffer may still be read or written on the stream
    cudaFree(c->d_stage);
    c->d_stage = p; c->stage_cap = cap;
    return 0;
}

struct PassArgs {
    jpeg::Quant qt;
    int W, H, mcux, mcuy, seg_words;
    long mcus, nf;
    const unsigned char *rgb;                 // the pass's first frame
    int16_t *coef;                            // [nf][mcus][6][64] zigzag
    uint32_t *words;                          // [nf * mcuy][seg_words] big-endian bit stream of each segment
    int *seg_raw, *seg_len;                   // [nf * mcuy] bytes before / after stuffing
    size_t *seg_off, *fsize, *foff;           // [nf * mcuy] offset in its frame; [nf] frame bytes; [nf] frame offset in out
    const uint8_t *hdr;
    unsigned char *out;
};

__global__ void __launch_bounds__(128) k_jpeg_blocks(const __grid_constant__ PassArgs a) {
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a.mcus * jpeg::BLK) return;
    const long m = i / jpeg::BLK;
    const int b = (int)(i - m * jpeg::BLK), mx = (int)(m % a.mcux), my = (int)(m / a.mcux);
    for (long f = blockIdx.y; f < a.nf; f += gridDim.y)
        jpeg::encode_block(a.rgb + (size_t)f * a.H * a.W * 3, a.W, a.H, mx, my, b, a.qt, a.coef + ((size_t)f * a.mcus * jpeg::BLK + i) * 64);
}

// ORs (bits, len) into a segment's big-endian words at bit position pos
struct EmitBits {
    uint32_t *w;
    unsigned pos;
    __device__ void operator()(unsigned v, int len) {
        if (len == 0) return;
        const unsigned k = pos >> 5, o = pos & 31;
        if (o + len <= 32) atomicOr(w + k, v << (32 - o - len));
        else { atomicOr(w + k, v >> (o + len - 32)); atomicOr(w + k + 1, v << (64 - o - len)); }
        pos += len;
    }
};

__global__ void __launch_bounds__(ROW_WARPS * 32) k_jpeg_rows(const __grid_constant__ PassArgs a) {
    const int lane = threadIdx.x & 31, row = blockIdx.x * ROW_WARPS + (threadIdx.x >> 5);
    if (row >= a.mcuy) return;                                      // a whole warp: nothing below synchronises the block
    const int nb = a.mcux * jpeg::BLK;
    for (long f = blockIdx.y; f < a.nf; f += gridDim.y) {
        const size_t seg = (size_t)f * a.mcuy + row;
        uint32_t *wd = a.words + seg * a.seg_words;
        const int16_t *cf = a.coef + ((size_t)f * a.mcus + (size_t)row * a.mcux) * jpeg::BLK * 64;
        unsigned carry = 0;
        for (int base = 0; base < nb; base += 32) {
            const int i = base + lane, mx = i / jpeg::BLK, b = i - mx * jpeg::BLK;
            int pred = 0, bits = 0;
            if (i < nb) {
                const int p = jpeg::prev_block(mx, b);
                pred = p < 0 ? 0 : cf[(size_t)p * 64];
                jpeg::CountBits cb;
                jpeg::code_block(cf + (size_t)i * 64, pred, c_tab, b < 4 ? 0 : 2, cb);
                bits = cb.n;
            }
            int incl = bits;
            for (int d = 1; d < 32; d <<= 1) {
                const int v = __shfl_up_sync(0xffffffffu, incl, d);
                if (lane >= d) incl += v;
            }
            const unsigned total = (unsigned)__shfl_sync(0xffffffffu, incl, 31);
            // the words this chunk starts: the first one may hold the previous chunk's last bits
            for (unsigned w = ((carry + 31) >> 5) + lane; w < ((carry + total + 31) >> 5); w += 32) wd[w] = 0;
            __syncwarp();
            if (i < nb) {
                EmitBits e{wd, carry + (unsigned)(incl - bits)};
                jpeg::code_block(cf + (size_t)i * 64, pred, c_tab, b < 4 ? 0 : 2, e);
            }
            __syncwarp();
            carry += total;
        }
        const unsigned pad = (8 - (carry & 7)) & 7;                // 1-bits to the byte boundary: the word already holds bits
        if (lane == 0 && pad) atomicOr(wd + (carry >> 5), ((1u << pad) - 1) << (32 - (carry & 31) - pad));
        __syncwarp();
        const int raw = (int)((carry + pad) >> 3);
        int ff = 0;
        for (int k = lane; k < raw; k += 32) ff += ((wd[k >> 2] >> (24 - 8 * (k & 3))) & 255u) == 255u;
        for (int d = 16; d; d >>= 1) ff += __shfl_xor_sync(0xffffffffu, ff, d);
        if (lane == 0) { a.seg_raw[seg] = raw; a.seg_len[seg] = raw + ff; }
    }
}

__global__ void k_jpeg_frame(const __grid_constant__ PassArgs a) {
    const long f = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= a.nf) return;
    size_t o = jpeg::HEADER_BYTES;
    for (int r = 0; r < a.mcuy; r++) {
        const size_t seg = (size_t)f * a.mcuy + r;
        a.seg_off[seg] = o;
        o += (size_t)a.seg_len[seg] + (r + 1 < a.mcuy ? 2 : 0);
    }
    a.fsize[f] = o + 2;
}

__global__ void __launch_bounds__(32) k_jpeg_write(const __grid_constant__ PassArgs a) {
    const int lane = threadIdx.x, r = blockIdx.x;
    for (long f = blockIdx.y; f < a.nf; f += gridDim.y) {
        unsigned char *o = a.out + a.foff[f];
        const size_t seg = (size_t)f * a.mcuy + r, off = a.seg_off[seg];
        if (r == 0) for (int k = lane; k < jpeg::HEADER_BYTES; k += 32) o[k] = a.hdr[k];
        if (lane == 0 && r > 0) { o[off - 2] = 0xFF; o[off - 1] = (unsigned char)(0xD0 + ((r - 1) & 7)); }
        if (lane == 0 && r == a.mcuy - 1) { o[off + a.seg_len[seg]] = 0xFF; o[off + a.seg_len[seg] + 1] = 0xD9; }
        const uint32_t *wd = a.words + seg * a.seg_words;
        const int raw = a.seg_raw[seg];
        size_t pos = off;
        for (int base = 0; base < raw; base += 32) {
            const int k = base + lane;
            const unsigned byte = k < raw ? (wd[k >> 2] >> (24 - 8 * (k & 3))) & 255u : 0u;
            const unsigned ffs = __ballot_sync(0xffffffffu, k < raw && byte == 255u);
            if (k < raw) {
                const size_t p = pos + lane + __popc(ffs & ((1u << lane) - 1));
                o[p] = (unsigned char)byte;
                if (byte == 255u) o[p + 1] = 0;
            }
            pos += (size_t)(raw - base < 32 ? raw - base : 32) + __popc(ffs);
        }
    }
}

unsigned frames_grid(long nf) { return (unsigned)(nf < 65535 ? nf : 65535); }

// blocks, rows and frame sizes of frames f0 .. f0 + nf - 1, the sizes on the host (synchronises the stream)
int encode_pass(PassArgs &a, const unsigned char *rgb, long f0, long nf, cudaStream_t st) {
    a.nf = nf;
    a.rgb = rgb + (size_t)f0 * a.H * a.W * 3;
    const unsigned gy = frames_grid(nf);
    k_jpeg_blocks<<<dim3((unsigned)((a.mcus * jpeg::BLK + 127) / 128), gy), 128, 0, st>>>(a);
    CK(cudaGetLastError());
    k_jpeg_rows<<<dim3((unsigned)((a.mcuy + ROW_WARPS - 1) / ROW_WARPS), gy), ROW_WARPS * 32, 0, st>>>(a);
    CK(cudaGetLastError());
    k_jpeg_frame<<<(unsigned)((nf + 127) / 128), 128, 0, st>>>(a);
    CK(cudaGetLastError());
    return 0;
}

int pass_sizes(const PassArgs &a, size_t *h_fsize, cudaStream_t st) {
    CK(cudaMemcpyAsync(h_fsize, a.fsize, (size_t)a.nf * sizeof(size_t), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    return 0;
}

}  // namespace

extern "C" {

size_t uhc_jpeg_bound(int W, int H) {
    if (W < 1 || H < 1 || W > jpeg::MAX_WH || H > jpeg::MAX_WH) return 0;
    return jpeg::frame_bound(W, H);
}

int uhc_jpeg_encode(UhcEngine *e, const unsigned char *rgb_dev, long n, int W, int H, int quality, unsigned char *out_dev, size_t out_cap,
                    size_t *offsets_dev, size_t *total_host, void *stream) {
    if (!e) { uhc_err() = "uhc_jpeg_encode: null engine"; return -2; }
    if (n < 0) { uhc_err() = "uhc_jpeg_encode: n < 0"; return -2; }
    if (W < 1 || H < 1 || W > jpeg::MAX_WH || H > jpeg::MAX_WH) { uhc_err() = "uhc_jpeg_encode: W and H must be in 1 .. 16384"; return -2; }
    if (quality < 1 || quality > 100) { uhc_err() = "uhc_jpeg_encode: quality must be in 1 .. 100"; return -2; }
    if (n > 0 && (!rgb_dev || !out_dev || !offsets_dev || !total_host)) { uhc_err() = "uhc_jpeg_encode: null pointer with n > 0"; return -2; }
    cudaStream_t st = (cudaStream_t)stream;
    if (n == 0) {
        if (total_host) *total_host = 0;
        if (offsets_dev) {
            const size_t zero = 0;
            CK(cudaMemcpyAsync(offsets_dev, &zero, sizeof(size_t), cudaMemcpyHostToDevice, st));
            CK(cudaStreamSynchronize(st));
        }
        return 0;
    }
    const Geometry g = geometry(W, H);
    const long per_pass = (long)(SCRATCH_CAP / frame_scratch(g));
    const long pf = per_pass < 1 ? 1 : per_pass < n ? per_pass : n;
    VideoCtx *c = get_ctx(e);
    if (int rc = reserve(c, g, pf, st)) return rc;
    PassArgs a;
    jpeg::make_quant(quality, a.qt);
    uint8_t hdr[jpeg::HEADER_BYTES];
    jpeg::make_header(W, H, a.qt, hdr);
    jpeg::Tables tab;
    jpeg::make_tables(tab);
    CK(cudaMemcpyToSymbolAsync(c_tab, &tab, sizeof(tab), 0, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(c->d_hdr, hdr, sizeof(hdr), cudaMemcpyHostToDevice, st));
    a.W = W; a.H = H; a.mcux = g.mcux; a.mcuy = g.mcuy; a.seg_words = g.seg_words; a.mcus = g.mcus;
    a.coef = c->d_coef; a.words = c->d_words; a.seg_raw = c->d_seg_raw; a.seg_len = c->d_seg_len; a.seg_off = c->d_seg_off;
    a.fsize = c->d_fsize; a.foff = c->d_foff; a.hdr = c->d_hdr; a.out = out_dev;
    std::vector<size_t> offs((size_t)n + 1, 0);
    // one pass, or several into a buffer that holds n worst-case frames: written straight into out_dev.  Several passes that could overflow
    // out_cap: staged until the total is known (frames past out_cap are only sized).
    const bool single = pf == n, staged = !single && out_cap / (size_t)n < jpeg::frame_bound(W, H);
    for (long f0 = 0; f0 < n; f0 += pf) {
        const long nf = n - f0 < pf ? n - f0 : pf;
        if (int rc = encode_pass(a, rgb_dev, f0, nf, st)) return rc;
        if (int rc = pass_sizes(a, c->h_fsize, st)) return rc;
        for (long f = 0; f < nf; f++) offs[(size_t)(f0 + f) + 1] = offs[(size_t)(f0 + f)] + c->h_fsize[f];
        const size_t end = offs[(size_t)(f0 + nf)];
        if (end > out_cap) continue;                                // -3 below: sized, nothing written
        if (staged) {
            if (int rc = reserve_stage(c, end, offs[(size_t)f0], out_cap, st)) return rc;
            a.out = c->d_stage;
        }
        CK(cudaMemcpyAsync(c->d_foff, offs.data() + f0, (size_t)nf * sizeof(size_t), cudaMemcpyHostToDevice, st));
        k_jpeg_write<<<dim3((unsigned)g.mcuy, frames_grid(nf)), 32, 0, st>>>(a);
        CK(cudaGetLastError());
    }
    if (offs[(size_t)n] > out_cap) {
        *total_host = offs[(size_t)n];
        uhc_err() = "uhc_jpeg_encode: out_cap " + std::to_string(out_cap) + " < the " + std::to_string(offs[(size_t)n]) + " bytes of the frames";
        return -3;
    }
    if (staged) CK(cudaMemcpyAsync(out_dev, c->d_stage, offs[(size_t)n], cudaMemcpyDeviceToDevice, st));
    CK(cudaMemcpyAsync(offsets_dev, offs.data(), ((size_t)n + 1) * sizeof(size_t), cudaMemcpyHostToDevice, st));
    CK(cudaStreamSynchronize(st));
    *total_host = offs[(size_t)n];
    return 0;
}

void uhc_video_release(UhcEngine *e) {
    VideoCtx *c = e ? (VideoCtx *)engine_slot(e, SLOT_VIDEO) : nullptr;
    if (!c) return;
    cudaFree(c->d_coef); cudaFree(c->d_words); cudaFree(c->d_seg_raw); cudaFree(c->d_seg_len); cudaFree(c->d_seg_off);
    cudaFree(c->d_fsize); cudaFree(c->d_foff); cudaFreeHost(c->h_fsize); cudaFree(c->d_hdr); cudaFree(c->d_stage);
    delete c; engine_slot(e, SLOT_VIDEO) = nullptr;
}

}  // extern "C"
