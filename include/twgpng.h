/* twgpng.h -- C ABI of the PNG decoder in libtwg.so, the PNG half of image translation's decoding front end.
 *
 * Kept apart from include/twg.h, the ABI of the training and inference kernels, as include/twgjpeg.h is: these entries
 * belong to file input, not to the model, and twingan_b200/_lib.py binds them from this header under their own prefix,
 * `twgpng_`.  The conventions of twg.h hold: device pointers owned by the caller, no allocation at run time, asynchronous
 * on the given cudaStream_t and graph-capturable, 0 on success and < 0 on an invalid argument or CUDA error
 * (twg_last_error).
 */
#ifndef TWGPNG_H_
#define TWGPNG_H_

#include "twg.h"

#ifdef __cplusplus
extern "C" {
#endif
/* ---- PNG decoding into the uint8 payload of twg_images_u8_to_batch (util_io.imread's PIL decode of a PNG file): inflate
 *      (RFC 1950 / 1951) with the Adler-32 check, unfiltering, and the expansion to RGB of PIL's convert('RGB').  PNG is
 *      lossless, so the pixels equal PIL's.  The host (twingan_b200/png.py) reads the chunks, keeps the files this path
 *      decodes (no interlace, no APNG, no palette tRNS, known chunks only, every CRC right) and packs, per image, one
 *      int64 row of
 *        images [nimages][12] {stream start, stream end, inflated offset, inflated bytes, payload byte offset, H, W, colour
 *                              type, bit depth, row bytes, palette row (-1: none), first pixel}:
 *                              data[start, end) is the image's zlib stream (its IDAT payloads back to back); the stream
 *                              inflates into raw[offset, offset + H * (1 + row bytes)); first pixel = sum of H * W of the
 *                              images before it;
 *        palettes [rows][768] uint8 RGB, zero past each PLTE's entries (PIL maps an index past them to black).
 *      status: int32 [nimages], the OR of the TWG_PNG_* bits below (0: decoded exactly).  A flagged image's output is
 *      undefined: decode it again on the host.  A stream reads only data[start, end) and writes only its own region,
 *      whatever its bytes. */
#define TWG_PNG_HEADER 1         /* zlib header: CM != 8, CINFO > 7, FCHECK, or FDICT set */
#define TWG_PNG_BLOCK 2          /* block type 3, or a stored block with LEN != ~NLEN */
#define TWG_PNG_CODES 4          /* over-subscribed or incomplete code set, too many symbols, a bad repeat */
#define TWG_PNG_SYMBOL 8         /* a code of no symbol, or an invalid literal/length or distance symbol */
#define TWG_PNG_DISTANCE 16      /* a distance before the start of the output or beyond the declared window */
#define TWG_PNG_TRUNCATED 32     /* the stream ended before its final block and Adler-32 trailer */
#define TWG_PNG_LONG 64          /* the stream inflates to more than H * (1 + row bytes) */
#define TWG_PNG_SHORT 128        /* ... or to fewer bytes */
#define TWG_PNG_TRAILING 256     /* bytes after the zlib stream */
#define TWG_PNG_ADLER 512        /* the Adler-32 trailer does not match the inflated bytes */
#define TWG_PNG_FILTER 1024      /* a row's filter type is > 4 */
/* inflate and Adler-32, one warp per image, into raw; resets status[0..nimages) first. */
int twgpng_inflate(const void* data, const int64_t* images, int nimages, void* raw, void* status, twg_stream_t stream);
/* unfiltering (None / Sub / Up / Average / Paeth at the pixel's byte distance, 1 for sub-byte depths) of every row, in
 * place in raw, one CTA per image; skips flagged images and ORs TWG_PNG_FILTER into status. */
int twgpng_unfilter(void* raw, const int64_t* images, int nimages, void* status, twg_stream_t stream);
/* PIL's convert('RGB') of the unfiltered rows into payload (uint8 HWC at each image's offset), one thread per pixel;
 * npixels = sum of H * W.  Grey scales 1 / 2 / 4-bit samples to 0..255 and takes min(v, 255) of 16-bit ones; RGB,
 * grey+alpha and RGBA take the high byte of 16-bit samples and drop alpha; palette indices look up `palettes`. */
int twgpng_rgb(const void* raw, const int64_t* images, int nimages, const void* palettes, int64_t npixels,
               const void* status, void* payload, twg_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* TWGPNG_H_ */
