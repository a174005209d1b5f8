/* twgjpegp.h -- C ABI of the progressive JPEG entropy decoder in libtwg.so, the image-decoding front end of image
 * translation.
 *
 * A progressive file whose every coefficient is refined to its last bit decodes, in libjpeg, to the pixels of a baseline
 * file with the same coefficients: only the entropy decoding differs.  These entries fill the coefficient blocks; the
 * baseline entries twgjpeg_idct and twgjpeg_color of twgjpeg.h turn them into pixels.  Bound by twingan_b200/_lib.py
 * under the prefix `twgjpegp_`; the conventions of twg.h hold: device pointers owned by the caller, no allocation at run
 * time, asynchronous on the given cudaStream_t and graph-capturable, 0 on success and < 0 on an invalid argument or CUDA
 * error (twg_last_error).
 *
 * The host (twingan_b200/jpeg_progressive.py) parses the file, keeps the progressions this path restates and packs:
 *   segs   [nseg][6]   {byte start, byte end, scan row, first MCU, MCU count, marker}: one entropy-coded segment (a
 *                      restart interval of a scan, or the whole scan) at data[start, end); data[end], data[end + 1] must
 *                      be FF `marker` (RSTn in sequence from RST0 in every scan; after a scan's last segment, the marker
 *                      that ends the scan, EOI after the last scan);
 *   scans  [nscan][16] {image, Ss, Se, Ah, Al, components in the scan (1..3), their comp rows[3], their Huffman table
 *                      rows[3] (DC for a DC first scan, AC for an AC scan, -1 for a DC refinement), MCUs wide (an
 *                      interleaved scan: the frame's MCUs; one component: that component's blocks, one per MCU),
 *                      restart interval, level, 0};
 *   comps, images, qt, huff as twgjpeg.h describes them (twgjpeg_idct and twgjpeg_color read them unchanged).
 * coefs: int16 [blocks][64] zig-zag, as twgjpeg_entropy writes them.  Scans are grouped in levels: the scans of one level
 * write disjoint coefficients and read only what earlier levels wrote, so each level is one launch, in stream order.
 * status: int32 [nimages], the OR of the TWG_JPEG_* bits of twgjpeg.h and the bits below (0: decoded exactly).  A flagged
 * image's output is undefined: decode it again on the host. */
#ifndef TWGJPEGP_H_
#define TWGJPEGP_H_

#include "twgjpeg.h"

#ifdef __cplusplus
extern "C" {
#endif
#define TWG_JPEGP_REFINE_SIZE 64    /* an AC refinement symbol whose size is neither 0 nor 1 */
#define TWG_JPEGP_BAND 128          /* a coefficient written past the scan's Se */
#define TWG_JPEGP_VALUE_RANGE 256   /* a coefficient outside int16: s << Al, or a correction of +-(1 << Al) */
/* zero coefs[0 .. nblocks * 64) and status[0 .. nimages): progressive scans only add to the blocks.  coefs 16-byte
 * aligned. */
int twgjpegp_reset(void* coefs, int64_t nblocks, void* status, int nimages, twg_stream_t stream);
/* entropy decoding of the nseg segments of one level (T.81 G.1.2: DC first, DC refinement, AC first with end-of-band
 * runs, AC refinement with correction bits; DC predictions and end-of-band run reset at every restart), one thread per
 * segment, into coefs. */
int twgjpegp_entropy(const void* data, const int64_t* segs, int nseg, const int64_t* scans, const int64_t* comps,
                     const void* huff, void* coefs, void* status, twg_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* TWGJPEGP_H_ */
