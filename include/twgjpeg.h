/* twgjpeg.h -- C ABI of the baseline JPEG decoder in libtwg.so, the image-decoding front end of image translation.
 *
 * Kept apart from include/twg.h, the ABI of the training and inference kernels: these entries belong to file input, not
 * to the model, and twingan_b200/_lib.py binds them from this header under their own prefix, `twgjpeg_`.  The
 * conventions of twg.h hold: device pointers owned by the caller, no allocation at run time, asynchronous on the given
 * cudaStream_t and graph-capturable, 0 on success and < 0 on an invalid argument or CUDA error (twg_last_error).
 */
#ifndef TWGJPEG_H_
#define TWGJPEG_H_

#include "twg.h"

#ifdef __cplusplus
extern "C" {
#endif
/* ---- baseline JPEG decoding into the uint8 payload of twg_images_u8_to_batch (util_io.imread's PIL decode of a JPEG file), three stages whose result is
 *      bit for bit libjpeg-turbo's with its defaults (islow IDCT, fancy upsampling), as PIL calls it.  The host
 *      (twingan_b200/jpeg.py) parses the headers, keeps the files this path restates (SOF0 / 8-bit SOF1, one scan of every
 *      component, grey or YCbCr, 4:4:4 / 4:2:2 / 4:2:0) and packs the descriptors below (int64 rows):
 *        segs   [nseg][6]    {byte start, byte end, image, first MCU, MCU count, index of the segment in its image}: one
 *                            entropy-coded segment (a restart interval, or the whole scan) at data[start, end); data[end],
 *                            data[end + 1] must be FF D0+(index % 8), or FF D9 after the image's last segment;
 *        comps  [ncomps][10] {first block, blocks wide, blocks high, plane byte offset, quant row, DC table, AC table, h, v,
 *                            image}: one component's coefficient blocks (block-row-major from `first block`) and sample
 *                            plane (blocks wide * 8 bytes per row, 16-byte aligned offset), in image order, block ranges
 *                            ascending;
 *        images [nimages][12] {first comp row, comps (1 or 3), MCUs wide, H, W, payload byte offset, first pixel, segments,
 *                            hmax, vmax, 0, 0}: first pixel = sum of H * W of the images before it;
 *        qt     [rows][64] int32 quantisation tables in zig-zag order; huff [tables][1024] int32 Huffman tables, each
 *                            lut[512] (length << 8 | symbol for every code of <= 9 bits, indexed by the next 9 bits; 0 for
 *                            longer codes) | maxcode[18] (index = length; -1 when none) | valoff[18] | vals[256] | pad.
 *      coefs: int16 [blocks][64] zig-zag, DC-predicted; planes: uint8 sample planes; status: int32 [nimages], the OR of the
 *      TWG_JPEG_* bits below (0: decoded exactly).  A flagged image's output is undefined: decode it again on the host. */
#define TWG_JPEG_BAD_CODE 1       /* a bit pattern that is no code of its Huffman table */
#define TWG_JPEG_MARKER 2         /* FF followed by anything but 00 inside a segment */
#define TWG_JPEG_TRUNCATED 4      /* the segment ended before its last MCU */
#define TWG_JPEG_RESTART 8        /* the marker after a segment is not the RSTn / EOI it should be */
#define TWG_JPEG_COEF_RANGE 16    /* a DC value outside int16, or a run past the 64th coefficient */
#define TWG_JPEG_IDCT_RANGE 32    /* a dequantised or first-pass value outside int16, or an output outside [-512, 511] */
/* entropy decoding, one thread per segment; resets status[0..nimages) first.  coefs 16-byte aligned. */
int twgjpeg_entropy(const void* data, const int64_t* segs, int nseg, const int64_t* images, int nimages,
                     const int64_t* comps, const void* huff, void* coefs, void* status, twg_stream_t stream);
/* dequantisation and islow inverse DCT (jidctint.c's integer algorithm and range limit), one thread per block, into the
 * planes; ORs TWG_JPEG_IDCT_RANGE into status.  coefs, qt, planes 16-byte aligned. */
int twgjpeg_idct(const void* coefs, const int64_t* comps, int ncomps, int64_t nblocks, const void* qt, void* planes,
                  void* status, twg_stream_t stream);
/* fancy h2v1 / h2v2 chroma upsampling (triangle filter, alternating rounding bias, last real column / row replicated;
 * replication for chroma planes of <= 2 columns) and jdcolor.c's fixed-point YCbCr -> RGB (grey repeated in the three
 * channels), uint8 HWC into payload at each image's offset; npixels = sum of H * W. */
int twgjpeg_color(const void* planes, const int64_t* images, int nimages, const int64_t* comps, int64_t npixels,
                   void* payload, twg_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* TWGJPEG_H_ */
