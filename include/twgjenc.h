/* twgjenc.h -- C ABI of the baseline JPEG encoder in libtwg.so, the image-encoding back end of image translation.
 *
 * Kept apart from include/twg.h (the model) and include/twgjpeg.h (the decoder): twingan_b200/_lib.py binds these
 * entries from this header under their own prefix, `twgjenc_`.  The conventions of twg.h hold: device pointers owned by
 * the caller, scratch sized by twgjenc_workspace_bytes, no allocation at run time, asynchronous on the given
 * cudaStream_t and graph-capturable, 0 on success and -1 on an invalid argument (twg_last_error).
 */
#ifndef TWGJENC_H_
#define TWGJENC_H_

#include "twg.h"

#ifdef __cplusplus
extern "C" {
#endif
/* ---- baseline JPEG encoding of n equal-size uint8 RGB images (HWC, [n][h][w][3]), byte for byte the scan libjpeg-turbo
 *      writes at PIL's defaults: 4:2:0 (Y 2x2, Cb and Cr 1x1), the islow forward DCT, libjpeg-turbo's reciprocal
 *      quantisation, the Annex K Huffman tables, no restart markers.  twingan_b200/jpeg.py writes the header around it.
 *      1 <= h, w <= 65535 and h * w <= 2^25.  An image has mx * my MCUs, mx = ceil(w / 16), my = ceil(h / 16), and
 *      6 * mx * my coded blocks in MCU order, each MCU Y00 Y01 Y10 Y11 Cb Cr (dummy blocks fill a partial MCU).
 *        qt     int32 [2][64]: the luma and chroma quantisation tables in zig-zag order, values 4..255 (so every DC
 *               difference and AC value has an Annex K symbol; jpeg.encoder_qt's quality-75 tables qualify);
 *        coefs  int16 [n][blocks][64]: quantised coefficients in zig-zag order, DC not predicted;
 *        bitpos int32 [n][blocks + 1]: per image, the exclusive prefix sum of the blocks' code lengths in bits (the last
 *               entry is the image's scan length before padding);
 *        out    the n scans back to back, each padded with 1 bits to a byte and 0xFF-stuffed, without markers; holds
 *               twgjenc_scan_capacity bytes;
 *        offsets int64 [n + 1]: image i's scan is out[offsets[i], offsets[i + 1]). */
int64_t twgjenc_workspace_bytes(int n, int h, int w);
int64_t twgjenc_scan_capacity(int n, int h, int w);
/* colour conversion (jccolor.c), edge expansion (jcsample.c, jcprepct.c), h2v2 downsampling, islow forward DCT and
 * quantisation, one thread per block.  coefs 16-byte aligned. */
int twgjenc_dct(const void* rgb, int n, int h, int w, const void* qt, void* coefs, twg_stream_t stream);
/* the Huffman code length of every block (DC predicted per component in MCU order from 0) and its prefix sum per image,
 * one CTA per image.  coefs 16-byte aligned. */
int twgjenc_bits(const void* coefs, int n, int h, int w, void* bitpos, twg_stream_t stream);
/* the codes of every block written at its bit position, the padding, then 0xFF stuffing and packing of the scans back to
 * back with their offsets.  coefs, workspace 16-byte aligned. */
int twgjenc_pack(const void* coefs, const void* bitpos, int n, int h, int w, void* workspace, void* out, void* offsets,
                 twg_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* TWGJENC_H_ */
