/* uhc_video.h -- C ABI of the batched JPEG encoder (part of libuhc_b200.so): the renderer's frames compressed on the GPU, so that only the
 * compressed bytes leave the device.
 *
 * One fixed format: baseline sequential JPEG (ITU-T T.81) in a JFIF file, full-range BT.601 YCbCr, 4:2:0 subsampling, the Annex K quantisation
 * tables scaled by quality as IJG does, the four Annex K Huffman tables, and a restart interval of one MCU row (RST0 .. RST7 between the rows).
 * The arithmetic is integer throughout (uhc_b200/csrc/video_core.h), so the bytes do not depend on the device.  Pointers suffixed _dev are
 * CUDA device pointers; byte counts and offsets are size_t.
 */
#ifndef UHC_VIDEO_H
#define UHC_VIDEO_H
#include <stddef.h>
#include "uhc_b200.h"
#ifdef __cplusplus
extern "C" {
#endif

/* The most bytes one W x H frame can take, for any pixels and any quality (0 for W or H outside 1 .. 16384). */
size_t uhc_jpeg_bound(int W, int H);

/* n frames rgb_dev = [n][H][W][3] uint8 -> n JPEG files packed back to back in out_dev: file i is out_dev[offsets_dev[i] .. offsets_dev[i + 1]),
 * offsets_dev = [n + 1], *total_host = offsets_dev[n].  Synchronises `stream`.  Returns 0; -2 with nothing launched on a bad argument (a null
 * engine, n < 0, W or H outside 1 .. 16384, quality outside 1 .. 100, a null pointer with n > 0); -3 when out_cap is smaller than the total,
 * with *total_host set to it and nothing written to out_dev or offsets_dev; -1 on a CUDA error (uhc_last_error()).  Every frame is encoded
 * once.  Scratch of at most 256 MiB (or one frame, if a frame needs more) is kept per engine until uhc_video_release; a call of more frames than
 * that scratch holds, with out_cap < n * uhc_jpeg_bound(W, H), also keeps its files in a staging buffer of at most out_cap bytes until it knows
 * they fit, and copies them to out_dev then. */
int uhc_jpeg_encode(UhcEngine *e, const unsigned char *rgb_dev, long n, int W, int H, int quality, unsigned char *out_dev, size_t out_cap,
                    size_t *offsets_dev, size_t *total_host, void *stream);

/* Frees the encoder's scratch of this engine (also safe without any); optional: uhc_engine_destroy frees it too. */
void uhc_video_release(UhcEngine *e);

#ifdef __cplusplus
}
#endif
#endif
