/*
 * b200jpg.h -- the C ABI of the H100-native baseline-JPEG decode path.
 *
 * This is the drop-in boundary beneath the reference's C++ interface (include/interface/jpeg.hpp restates
 * thorfdbg/libjpeg's interface/jpeg.hpp:79-250): plain pointers and sizes, no C++ and no torch types.
 * The C++ `class JPEG` shim (libjpeg_b200/csrc/jpeg_shim.cpp) calls these entry points (and, for device bitmaps, the
 * library's internal rectangle-to-bitmap copy kernel); the batch
 * entry points are what the throughput benchmark and the Python host layer bind (ctypes).
 *
 * What each entry point replaces in the reference (file:line relative to the reference tree):
 *   b200jpg_parse            Decoder::ParseHeaderIncremental            codestream/decoder.cpp:77
 *                            Tables::ParseTablesIncremental             codestream/tables.cpp:1003-1420
 *                            Frame::ParseMarker / Scan::ParseMarker     marker/frame.cpp:111, marker/scan.cpp:163
 *                            EntropyParser::ParseRestartMarker (index)  codestream/entropyparser.cpp:117-136
 *   b200jpg_batch_decode     SequentialScan::ParseMCU / DecodeBlock     codestream/sequentialscan.cpp:381,678
 *     (entropy stage)        HuffmanDecoder::Get, BitStream<false>      coding/huffmandecoder.hpp:103, io/bitstream.cpp:56
 *     (reconstruction stage) BlockBitmapRequester::ReconstructRegion    control/blockbitmaprequester.cpp:1249
 *                            IDCT::InverseTransformBlock                dct/idct.cpp:226
 *                            Upsampler<sx,sy>::UpsampleRegion           upsampling/upsampler.cpp:83
 *                            YCbCrTrafo::YCbCr2RGB                      colortrafo/ycbcrtrafo.cpp:679
 *   b200jpg_batch_decode_into  the same, into per-component ImageBitMaps interface/imagebitmap.hpp:104-109
 *   b200jpg_batch_decode_into_ex  the same, samples converted to float32 / float16 / bfloat16 on the way out (no counterpart)
 *   b200jpg_batch_decode_into_table  the same, every sample looked up in a per-component table (no counterpart)
 *   b200jpg_last_error       JPEG::LastError                            interface/jpeg.cpp:962
 *
 * Error codes are the reference's (interface/parameters.hpp:1156-1228).
 * There is NO CPU fallback: every decode entry point fails with B200JPG_ERR_NO_DEVICE when no CUDA device
 * is usable.
 */
#ifndef B200JPG_H
#define B200JPG_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#ifndef B200JPG_API
#define B200JPG_API __attribute__((visibility("default")))
#endif

#define B200JPG_OK 0
#define B200JPG_ERR_INVALID_PARAMETER (-1024)
#define B200JPG_ERR_UNEXPECTED_EOF (-1025)
#define B200JPG_ERR_OBJECT_DOESNT_EXIST (-1031)
#define B200JPG_ERR_NOT_IMPLEMENTED (-1034)
#define B200JPG_ERR_MALFORMED_STREAM (-1038)
#define B200JPG_ERR_OUT_OF_MEMORY (-2048)
#define B200JPG_ERR_NO_DEVICE (-8193) /* in the reference's USER_ERROR range (-8192 and below) */
#define B200JPG_ERR_CUDA (-8194)

#define B200JPG_MAX_COMPONENTS 4
#define B200JPG_MAX_SCANS 16

/* Geometry of one parsed codestream (host only, no GPU needed). */
typedef struct b200jpg_frame_info {
    uint32_t width, height;
    uint8_t ncomp, precision, frame_type /* 0 = SOF0, 1 = SOF1, 2 = SOF2 (progressive) */, ycbcr /* 1: YCbCr->RGB applies */;
    uint8_t comp_id[B200JPG_MAX_COMPONENTS];
    uint8_t hs[B200JPG_MAX_COMPONENTS], vs[B200JPG_MAX_COMPONENTS];     /* sampling factors of the SOF */
    uint8_t subx[B200JPG_MAX_COMPONENTS], suby[B200JPG_MAX_COMPONENTS]; /* hmax/hs, vmax/vs (reference's SubX/SubY) */
    uint8_t tq[B200JPG_MAX_COMPONENTS];
    uint32_t mcu_cols, mcu_rows;                                       /* interleaved MCU grid */
    uint32_t blocks_w[B200JPG_MAX_COMPONENTS], blocks_h[B200JPG_MAX_COMPONENTS]; /* MCU-padded block grid */
    uint32_t nscans;
    uint32_t restart_interval;  /* DRI in effect at the first scan, MCUs; 0 = none */
    uint32_t n_intervals;       /* restart intervals over all scans */
    uint64_t ecs_bytes;         /* entropy coded bytes over all scans, as stored (stuffing + RSTn included) */
    uint64_t stored_blocks;     /* sum_c ceil(ceil(W/subx)/8)*ceil(ceil(H/suby)/8): the reference's block store */
} b200jpg_frame_info;

/* --- host-side parse, no device ------------------------------------------------------------------ */
/* Parses the marker segments of one codestream. Returns B200JPG_OK or a negative error code. */
B200JPG_API int b200jpg_parse(const uint8_t *data, size_t len, b200jpg_frame_info *info);
/* The Exif orientation 1..8 that B200JPG_FLAG_EXIF_ORIENTATION applies to this codestream (1 without a valid Exif orientation),
 * or the negative error code b200jpg_parse returns for it. Host only, no device. */
B200JPG_API int b200jpg_exif_orientation(const uint8_t *data, size_t len);
/* The colour space the output modes (B200JPG_FLAG_OUTPUT_RGB / _L, DESIGN §14 and §15) read a codestream's samples in. One
 * component: GREY. Three: YCBCR when b200jpg_frame_info::ycbcr is 1, else RGB. Four, 8-bit, with an APP14 segment in front of the
 * first scan whose payload has at least 12 bytes and starts with "Adobe" (the last such segment counts, libjpeg's examine_app14):
 * CMYK when its transform byte (payload[11]) is 0, YCCK for any other value (libjpeg's default_decompress_parms). Anything else --
 * two components, a four-component frame without such a segment or of 12 bits -- is UNKNOWN: a mode gives such a frame the status
 * B200JPG_ERR_NOT_IMPLEMENTED. Returns one of B200JPG_COLORSPACE_*, or the negative error code b200jpg_parse returns for it. Host
 * only, no device. */
#define B200JPG_COLORSPACE_UNKNOWN 0
#define B200JPG_COLORSPACE_GREY 1
#define B200JPG_COLORSPACE_YCBCR 2
#define B200JPG_COLORSPACE_RGB 3
#define B200JPG_COLORSPACE_CMYK 4
#define B200JPG_COLORSPACE_YCCK 5
B200JPG_API int b200jpg_colorspace(const uint8_t *data, size_t len);

/* Builds the device-independent Huffman / quantisation table blob of scan `scan` of one codestream on the host
 * (replaces HuffmanTemplate::BuildDecoder coding/huffmantemplate.cpp:802-874 and IDCT::DefineQuant dct/idct.cpp:98-108).
 * Returns the blob size (also when dst is NULL or too small), 0 on error. This blob is what rank 0 broadcasts. */
B200JPG_API uint64_t b200jpg_build_tables(const uint8_t *data, size_t len, int scan, uint8_t *dst, uint64_t capacity);

/* --- device context -------------------------------------------------------------------------------- */
typedef struct b200jpg_ctx b200jpg_ctx;

/* Creates a decode context on CUDA device `device` (current device if < 0). */
B200JPG_API int b200jpg_create(int device, b200jpg_ctx **ctx);
B200JPG_API void b200jpg_destroy(b200jpg_ctx *ctx);
/* Frees the device / pinned buffers the context keeps for reuse by later batches (buffers of live batches are untouched). */
B200JPG_API void b200jpg_trim(b200jpg_ctx *ctx);
/* Message and code of the last failure on this context (code 0 / "" when none). ctx may be NULL for
 * failures of b200jpg_create / b200jpg_parse on the calling thread. */
B200JPG_API int b200jpg_last_error(b200jpg_ctx *ctx, const char **message);

/* --- batches --------------------------------------------------------------------------------------- */
typedef struct b200jpg_batch b200jpg_batch;

/* Host stage: parses `n` codestreams (host pointers), builds the restart-interval index and the table
 * sets, and packs everything the kernels need into pinned staging memory.  Output layout: frame i is
 * written at out + out_offset(i) as interleaved 8-bit pixels, ncomp bytes per pixel, row pitch
 * width*ncomp (the layout a BitMapHook client with BytesPerPixel = depth gets from the reference).
 * Frames that fail to parse make the call fail unless `tolerate_bad` is non-zero, in which case they are
 * skipped and reported through b200jpg_batch_frame_status. */
B200JPG_API int b200jpg_batch_create(b200jpg_ctx *ctx, const uint8_t *const *frames, const size_t *lens, int n, int tolerate_bad,
                         b200jpg_batch **batch);
/* The same with request flags -- what a RectangleRequest carries besides the rectangle (codestream/rectanglerequest.cpp:
 * 93-165): B200JPG_FLAG_NO_COLOR_TRANSFORM = JPGTAG_MATRIX_LTRAFO set to JPGFLAG_MATRIX_COLORTRANSFORMATION_NONE: the
 * components are upsampled and delivered as they are (YCbCr frames come out as Y, Cb, Cr). */
#define B200JPG_FLAG_NO_COLOR_TRANSFORM 1u
/* B200JPG_FLAG_NO_UPSAMPLE = JPGTAG_DECODER_UPSAMPLE false (control/bitmapctrl.cpp:273-293, BlockBitmapRequester::
 * ReconstructUnsampled control/blockbitmaprequester.cpp:1013-1074): no upsampling and no colour transformation (the reference
 * refuses one without the other); frame i is written as plane after plane, component c holding ceil(width / subx[c]) x
 * ceil(height / suby[c]) samples, rows tightly packed.  Samples are bytes, or native-endian 16-bit for 12-bit frames. */
#define B200JPG_FLAG_NO_UPSAMPLE 2u
/* B200JPG_FLAG_DOWNSCALE_k (a two-bit field, B200JPG_FLAG_DOWNSCALE_MASK; no counterpart in the reference): every frame comes
 * out at W' = ceil(width / k) x H' = ceil(height / k). Each 8x8 block goes through a reduced inverse transform to
 * (8/k) x (8/k) samples -- the k x k box average of its exact IDCT, in fixed point as DESIGN §10 specifies -- and the result is
 * reconstructed like the IDCT output of a W' x H' frame with the same sampling factors: upsampling, colour transformation, clamp
 * and sample types as without the flag, B200JPG_FLAG_NO_COLOR_TRANSFORM and B200JPG_FLAG_NO_UPSAMPLE included (component c is
 * then ceil(W' / subx[c]) x ceil(H' / suby[c])). A frame's status is its status at full size; a JPEG XT frame with a residual
 * layer is B200JPG_ERR_NOT_IMPLEMENTED. Accepted by b200jpg_batch_create_ex, b200jpg_decode_to_host_ex and
 * b200jpg_decode_to_device_ex; these bits were ignored before they were defined. b200jpg_batch_output_extent gives the size. */
#define B200JPG_FLAG_DOWNSCALE_2 0x4u
#define B200JPG_FLAG_DOWNSCALE_4 0x8u
#define B200JPG_FLAG_DOWNSCALE_8 0xCu
#define B200JPG_FLAG_DOWNSCALE_MASK 0xCu
/* B200JPG_FLAG_EXIF_ORIENTATION (no counterpart in the reference, which skips the Exif segment): every frame leaves the decoder
 * as its oriented image. D is the image as it is written without the flag ([H, W, ...], after downscaling, colour transformation
 * and clamp; with B200JPG_FLAG_NO_UPSAMPLE each plane at its own extent), O what is written with it:
 *     1  D                       2  D mirrored left-right     3  D rotated by 180 deg     4  D mirrored top-bottom
 *     5  D transposed            6  D rotated 90 deg clockwise  7  D transposed about the anti-diagonal  8  D rotated 90 deg ccw
 * (PIL's ImageOps.exif_transpose). Width and height are swapped for 5..8: b200jpg_batch_output_extent, out_bytes / out_offset
 * and the descriptors of b200jpg_batch_decode_into(_ex) describe the oriented image. The orientation is tag 0x0112 of IFD0 of the
 * first APP1 segment in front of the first scan whose payload starts with "Exif\0\0" (b200jpg_exif_orientation); a malformed
 * segment means orientation 1 and never changes a frame's status or a sample. Accepted by b200jpg_batch_create_ex,
 * b200jpg_decode_to_host_ex and b200jpg_decode_to_device_ex. b200jpg_batch_decode_into(_ex) also refuses a frame of orientation 5..8
 * whose |bytes_per_row| exceeds INT32_MAX (it becomes that frame's pixel stride). b200jpg_batch_decode / b200jpg_batch_reconstruct
 * of a batch with oriented frames describe those frames' slots in a descriptor table like b200jpg_batch_decode_into's: each call
 * copies it to the device on the stream (one small H2D copy), and the host may wait for the copy issued three such calls earlier
 * before it reuses its pinned staging slot. Without oriented (or cropped, b200jpg_batch_create_crop) frames these calls stay as
 * before: no copy, no host wait. */
#define B200JPG_FLAG_EXIF_ORIENTATION 0x10u
/* Output modes (DESIGN §14; no counterpart in the reference): every frame of the batch leaves with the same number of components,
 * whatever it was coded with. B200JPG_FLAG_OUTPUT_RGB: 3 components. A 3-component frame is written as without the flag; a grey
 * frame's sample v goes to all three components (PIL's convert("RGB") of an L image), 8- and 12-bit alike.
 * B200JPG_FLAG_OUTPUT_L: 1 component. A grey frame is written as without the flag; a YCbCr frame (ycbcr == 1) as its component 0
 * with B200JPG_FLAG_NO_COLOR_TRANSFORM, the luma upsampled to the frame size (libjpeg's JCS_GRAYSCALE output) -- reconstructed
 * alone, its chroma entropy decoded but never transformed; a 3-component frame without colour transformation (ycbcr == 0) and a JPEG
 * XT frame after its merge as L = (19595 R + 38470 G + 7471 B + 32768) >> 16 of the clamped samples (PIL's convert("L")).
 * A CMYK or YCCK frame (b200jpg_colorspace; DESIGN §15) is converted as Pillow converts a four-component JPEG it reads as
 * Adobe-inverted CMYK: from the clamped samples s0..s3 written without the mode, a_c = 255 - s_c (CMYK), or a = R, G, B of libjpeg's
 * YCC -> RGB on s0, s1, s2 (YCCK), clamped; then out_c = s3 - MULDIV255(a_c, s3) with MULDIV255(a, b) = ((t >> 8) + t) >> 8,
 * t = a b + 128 (PIL's convert("RGB")), and under B200JPG_FLAG_OUTPUT_L the L formula of that RGB (PIL's convert("L")).
 * The mode is a per-pixel map between the colour transformation (and clamp) and the Exif orientation: the composition is
 * downscale -> mode -> orientation -> crop -> resize -> float map, whose scale[c] / bias[c] are those of the OUTPUT component c.
 * b200jpg_batch_output_extent (c below the output component count), out_bytes / out_offset (h x w x output components per slot)
 * and the descriptors of b200jpg_batch_decode_into(_ex) follow the output components (b200jpg_batch_output_components). A frame's
 * status is its status without the mode; a frame whose b200jpg_colorspace is B200JPG_COLORSPACE_UNKNOWN (2 components, 4 without
 * an Adobe segment or of 12 bits) has the status B200JPG_ERR_NOT_IMPLEMENTED (it fails the call, or with tolerate_bad it is
 * skipped). Both bits, or a mode bit with B200JPG_FLAG_NO_COLOR_TRANSFORM, is B200JPG_ERR_INVALID_PARAMETER for the call; a mode bit with B200JPG_FLAG_NO_UPSAMPLE is B200JPG_ERR_NOT_IMPLEMENTED. Accepted
 * wherever request flags are (b200jpg_output_size answers as without them). b200jpg_batch_decode / b200jpg_batch_reconstruct
 * describe the slots of the frames whose mode changes them like those of oriented frames: one small H2D copy per call. Without
 * either bit a batch is planned exactly as before. */
#define B200JPG_FLAG_OUTPUT_RGB 0x20u
#define B200JPG_FLAG_OUTPUT_L 0x40u
/* B200JPG_FLAG_LIBJPEG_TURBO (DESIGN §16; no counterpart in the reference): every frame is reconstructed as libjpeg-turbo (and so
 * Pillow) reconstructs it, in place of the reference's numerics, from the same dequantised coefficients:
 *   1. IDCT: libjpeg-turbo's JDCT_ISLOW in its C form with 64-bit intermediates. Constants (13 bits) 2446, 3196, 4433, 6270, 7373,
 *      9633, 12299, 15137, 16069, 16819, 20995, 25172; pass 1 down the columns descales by 11, (x + 2^10) >> 11, pass 2 along the
 *      rows by 18; the result v goes through the post-IDCT range-limit table at v & 1023 (0..127 -> v + 128, 128..511 -> 255,
 *      512..895 -> 0, 896..1023 -> v - 896): one uint8 plane per component.
 *   2. Upsampling of component c by fx = hmax / h_c, fy = vmax / v_c from its real size w x h = ceil(W h_c / hmax) x
 *      ceil(H v_c / vmax): 2x1 with w > 2: out[2j] = (3 a[j] + a[j-1] + 1) >> 2, out[2j+1] = (3 a[j] + a[j+1] + 2) >> 2,
 *      out[0] = a[0], out[2w-1] = a[w-1]; 1x2: upper (3 near + above + 1) >> 2, lower (3 near + below + 2) >> 2; 2x2 with w > 2:
 *      cs = 3 near + far (far: the row above for the upper output row, below for the lower), out[2j] = (3 cs[j] + cs[j-1] + 8) >> 4,
 *      out[2j+1] = (3 cs[j] + cs[j+1] + 7) >> 4, ends (4 cs[0] + 8) >> 4 and (4 cs[w-1] + 7) >> 4; any other integer ratio, and
 *      2x1 / 2x2 with w <= 2, replicates. The row above the first row and below row h - 1 is that row itself.
 *   3. Colour (b200jpg_colorspace YCbCr), b = Cb - 128, r = Cr - 128: R = Y + ((91881 r + 32768) >> 16), G = Y + ((-22554 b -
 *      46802 r + 32768) >> 16), B = Y + ((116130 b + 32768) >> 16), clamped to 0..255. RGB-coded frames: the identity; grey frames:
 *      the plane; B200JPG_FLAG_NO_COLOR_TRANSFORM: the upsampled components as they are.
 *   4. The output modes keep their meaning on these samples: B200JPG_FLAG_OUTPUT_L of a YCbCr frame is component 0 upsampled by
 *      rule 2 (Pillow's draft("L")), of an RGB-coded frame the L formula.
 *   5. A JPEG XT frame is its base codestream alone, as libjpeg-turbo decodes it. A JPEG XT frame whose profile the parser refuses
 *      (b200jpg_parse: B200JPG_ERR_NOT_IMPLEMENTED) keeps that status under the flag too: its base codestream is not decoded.
 *   6. With B200JPG_FLAG_OUTPUT_RGB or _L, a CMYK or YCCK frame (b200jpg_colorspace; DESIGN §18): its four components by rules 1
 *      and 2, then the conversion of B200JPG_FLAG_OUTPUT_RGB / _L for such frames (Pillow's convert("RGB") / convert("L") of the
 *      "CMYK" image it opens).
 * Everything after the reconstruction is unchanged (orientation, crop, resize, float map), as are extents, out_bytes and statuses.
 * The flag together with B200JPG_FLAG_DOWNSCALE_k or B200JPG_FLAG_NO_UPSAMPLE is B200JPG_ERR_NOT_IMPLEMENTED for the call; a 12-bit
 * frame, a two-component frame and a four-component frame without an output mode have the status B200JPG_ERR_NOT_IMPLEMENTED (it
 * fails the call, or with tolerate_bad it is skipped), as under a mode does a frame whose colorspace is
 * B200JPG_COLORSPACE_UNKNOWN. Accepted wherever request flags are. Without the flag a batch is planned exactly as before. libjpeg-turbo's reduced
 * decode at 1/2, 1/4 and 1/8 (Pillow's draft) is a per-frame request of b200jpg_batch_create_draft. */
#define B200JPG_FLAG_LIBJPEG_TURBO 0x80u
B200JPG_API int b200jpg_batch_create_ex(b200jpg_ctx *ctx, const uint8_t *const *frames, const size_t *lens, int n, int tolerate_bad,
                            unsigned flags, b200jpg_batch **batch);
/* A rectangle of a frame's output: columns x .. x + width - 1, rows y .. y + height - 1. {0, 0, 0, 0} is the whole frame. */
typedef struct b200jpg_rect {
    uint32_t x, y, width, height;
} b200jpg_rect;
/* b200jpg_batch_create_ex with a crop per frame (no counterpart in the reference). Let O be what the batch writes for the caller's
 * frame i without a crop, [H_o, W_o, C] after downscaling, colour transformation, clamp, Exif orientation and any float conversion
 * (b200jpg_batch_output_extent of the batch without rects). With rects[i] = (x, y, width, height), given in those output coordinates
 * (the composition is downscale -> orientation -> crop), frame i is written as exactly O[y : y + height, x : x + width], bit for
 * bit, for every destination kind, and nothing outside that rectangle's destination is written. b200jpg_batch_output_extent,
 * out_bytes / out_offset (the slot of a cropped frame holds width x height x C samples) and the descriptor rules of
 * b200jpg_batch_decode_into(_ex) then describe the cropped image. Every scan of every frame is still decoded in full, and a frame's
 * status is its status without the crop. The reconstruction runs only the tiles that cover the rectangle.
 * rects == NULL, or every entry {0, 0, 0, 0}: exactly b200jpg_batch_create_ex. Otherwise, for every frame that parses (the rectangle of
 * a frame that failed is ignored), a rectangle other than {0, 0, 0, 0} needs width >= 1, height >= 1, x + width <= W_o and
 * y + height <= H_o (in 64 bits); one that breaks this fails the call with B200JPG_ERR_INVALID_PARAMETER, tolerate_bad or not, and
 * the message names the frame. A rectangle together with B200JPG_FLAG_NO_UPSAMPLE is B200JPG_ERR_NOT_IMPLEMENTED for the call.
 * b200jpg_batch_decode / b200jpg_batch_reconstruct of a batch with cropped frames describe those frames' slots like those of oriented
 * frames: one small H2D copy per call (see B200JPG_FLAG_EXIF_ORIENTATION). */
B200JPG_API int b200jpg_batch_create_crop(b200jpg_ctx *ctx, const uint8_t *const *frames, const size_t *lens, int n, int tolerate_bad,
                                          unsigned flags, const b200jpg_rect *rects, b200jpg_batch **batch);
/* A target size of b200jpg_batch_create_resize. {0, 0}: the frame is not resized. */
typedef struct b200jpg_size {
    uint32_t width, height;
} b200jpg_size;
/* The filters of b200jpg_batch_create_resize, with the values of PIL's Image.Resampling (NEAREST, 0, is not one of them). */
#define B200JPG_RESAMPLE_LANCZOS 1
#define B200JPG_RESAMPLE_BILINEAR 2
#define B200JPG_RESAMPLE_BICUBIC 3
#define B200JPG_RESAMPLE_BOX 4
#define B200JPG_RESAMPLE_HAMMING 5
/* OpenCV's cv2.resize(C, (W_t, H_t), interpolation=INTER_LINEAR / INTER_AREA) instead of Pillow's resampler: 0x100 | cv2's own
 * constant (DESIGN §20). Every function that takes `resample` accepts them; with either, R below is cv2.resize of C, byte for
 * byte (OpenCV 4.13), and boxes and a reducing_gap are refused: B200JPG_ERR_INVALID_PARAMETER for the call, the frame named,
 * tolerate_bad or not. Windows, sizes, modes, orientation, drafts and the float map are as for Pillow's filters. An INTER_AREA
 * frame that shrinks by integer factors fx, fy with 255 fx fy >= 2^31 (OpenCV's int block sums overflow) is
 * B200JPG_ERR_NOT_IMPLEMENTED for the call. */
#define B200JPG_RESAMPLE_CV_LINEAR 0x101
#define B200JPG_RESAMPLE_CV_AREA 0x103
/* b200jpg_batch_create_crop with a target size per frame (no counterpart in the reference). Let C be what the batch writes for the
 * caller's frame i without a size: O[y : y + height, x : x + width] of b200jpg_batch_create_crop (O itself without a rectangle),
 * uint8, [h, w, ncomp]. With sizes[i] = {W_t, H_t}, frame i is written as R(C), bit for bit, where R is Pillow's convolution
 * resampler, Image.resize((W_t, H_t), resample) of a mode L / RGB / CMYK image (box=None, reducing_gap=None), applied to every
 * channel on its own: horizontal pass over the rows the vertical table touches, then vertical pass, in Pillow's 22-bit fixed
 * point; an axis whose size does not change is not resampled (DESIGN §13 states R exactly, including the one case where Pillow
 * runs the passes the other way round). A float destination of b200jpg_batch_decode_into_ex receives R(C) converted by its map:
 * the resize comes first. The composition is downscale -> orientation -> crop -> resize.
 * b200jpg_batch_output_extent, out_bytes / out_offset (the slot of a resized frame holds W_t x H_t x ncomp samples) and the
 * descriptor rules of b200jpg_batch_decode_into(_ex) then describe W_t x H_t, so one [N, C, H_t, W_t] tensor takes frames of any
 * size. A frame's status is its status without the size. Upscaling is allowed; a size too large to allocate is
 * B200JPG_ERR_OUT_OF_MEMORY (as is a side above 2^24 or W_t x H_t x ncomp above 2^34 bytes). The reconstruction writes C into a
 * scratch the batch owns, resized frames in reconstruction groups of their own, and two launches (two per 65535 resized frames)
 * resample it: a batch whose frames are all resized issues the launches of the same batch of b200jpg_batch_create_crop, with a
 * rectangle covering the whole output for a frame that has none, plus those two.
 * sizes == NULL, or every entry {0, 0}: exactly b200jpg_batch_create_crop (resample is then not looked at). Otherwise
 * B200JPG_ERR_INVALID_PARAMETER for the call, tolerate_bad or not, with the frame named in the message: a size with exactly one
 * zero field, or an unknown `resample`. A size together with B200JPG_FLAG_NO_UPSAMPLE is B200JPG_ERR_NOT_IMPLEMENTED for the call.
 * A 12-bit frame with a size has the status B200JPG_ERR_NOT_IMPLEMENTED: it fails the call, or with tolerate_bad it is skipped; it
 * is never written unresized. The size of a frame that fails to parse is ignored; a JPEG XT frame's residual codestream takes its
 * frame's size. b200jpg_batch_decode / b200jpg_batch_reconstruct of a batch with resized frames describe their slots like those of
 * cropped frames: one small H2D copy per call (see B200JPG_FLAG_EXIF_ORIENTATION). */
B200JPG_API int b200jpg_batch_create_resize(b200jpg_ctx *ctx, const uint8_t *const *frames, const size_t *lens, int n, int tolerate_bad,
                                            unsigned flags, const b200jpg_rect *rects, const b200jpg_size *sizes, int resample,
                                            b200jpg_batch **batch);
/* b200jpg_batch_create_resize with a requested size per frame for libjpeg-turbo's reduced decode, as Pillow's
 * JpegImageFile.draft(mode, (width, height)) asks for it (DESIGN §17; no counterpart in the reference). With drafts[i] = {w, h},
 * frame i of codestream size W x H is decoded at scale 1/k, k = b200jpg_draft_scale(frame, w, h), as ceil(W / k) x ceil(H / k), and
 * everything else follows on that image: the composition is draft -> mode -> orientation -> crop -> resize -> float map, rectangles
 * are given in the drafted, oriented image (b200jpg_output_size with B200JPG_FLAG_DOWNSCALE_k gives it) and a frame's status is its
 * status without the draft. At 1/k libjpeg-turbo's reconstruction (B200JPG_FLAG_LIBJPEG_TURBO rules 1-5) changes as follows, with
 * m = 8 / k and hmax, vmax the largest sampling factors:
 *   1. Component c is inverse transformed to s_c x s_c samples per block: s_c = m, doubled while s_c < 8, (hmax m) % (2 h_c s_c) == 0
 *      and (vmax m) % (2 v_c s_c) == 0 (jdmaster.c). s = 8: rule 1; 4: jpeg_idct_4x4; 2: jpeg_idct_2x2; 1: range_limit((F0 + 4) >>
 *      3) (jidctred.c, C form, 64-bit intermediates, then the range-limit table).
 *   2. Component c is upsampled by fx = hmax m / (h_c s_c), fy = vmax m / (v_c s_c) from its real size ceil(W' / fx) x ceil(H' / fy)
 *      of the reduced frame W' x H': by rule 2 for k = 2 and 4, replicated for k = 8 (libjpeg-turbo turns fancy upsampling off at
 *      1/8).
 * Both apply to all four components of a CMYK or YCCK frame under an output mode (rule 6), hmax and vmax over all four.
 * A frame whose k is 1 is decoded, planned and written exactly as without a draft. drafts == NULL, or every entry {0, 0}: exactly
 * b200jpg_batch_create_resize. Otherwise, for the call, tolerate_bad or not: an entry with exactly one zero field is
 * B200JPG_ERR_INVALID_PARAMETER (the message names the frame); a draft without B200JPG_FLAG_LIBJPEG_TURBO is
 * B200JPG_ERR_NOT_IMPLEMENTED, as B200JPG_FLAG_LIBJPEG_TURBO with B200JPG_FLAG_DOWNSCALE_k or B200JPG_FLAG_NO_UPSAMPLE stays. The
 * draft of a frame that fails to parse is ignored. */
B200JPG_API int b200jpg_batch_create_draft(b200jpg_ctx *ctx, const uint8_t *const *frames, const size_t *lens, int n, int tolerate_bad,
                                           unsigned flags, const b200jpg_size *drafts, const b200jpg_rect *rects, const b200jpg_size *sizes,
                                           int resample, b200jpg_batch **batch);
/* A source box of b200jpg_batch_create_resample, Pillow's Image.resize(box=(x0, y0, x1, y1)) in the coordinates of C (below).
 * {0, 0, 0, 0}: the default box (0, 0, w, h). */
typedef struct b200jpg_box {
    double x0, y0, x1, y1;
} b200jpg_box;
/* b200jpg_batch_create_draft with a source box and an output window per frame and one reducing_gap for the batch, the rest of
 * Pillow's Image.resize (DESIGN §19; no counterpart in the reference). Let C be what the batch writes for frame i without a size
 * (after draft, mode, orientation and crop, uint8, w x h). With sizes[i] = {W_t, H_t}, frame i is written, byte for byte, as
 *     Image.fromarray(C).resize((W_t, H_t), resample, box=box, reducing_gap=gap).crop((wx, wy, wx + ww, wy + wh))
 * of Pillow 12.2, where box = boxes[i] (the default box for {0, 0, 0, 0} or boxes == NULL), gap = reducing_gap (None when
 * reducing_gap <= 0) and (wx, wy, ww, wh) = windows[i] ({0, 0, 0, 0} or windows == NULL: the whole W_t x H_t image). That is:
 *   1. With a gap, fx = int((x1 - x0) / W_t / gap) or 1 and fy likewise, in double. If either is above 1, C is reduced over
 *      Pillow's _get_safe_box (the filter's support - 0.5 times the scale around the box, int() low, ceil() high, clamped to C) by
 *      Image.reduce: each fx x fy block (fewer pixels at the box's right and bottom edges) is ((s + n / 2) floor(2^24 / n)) >> 24
 *      for the sum s of its n pixels; the box becomes ((x0 - rx0) / fx, (y0 - ry0) / fy, (x1 - rx0) / fx, (y1 - ry0) / fy).
 *   2. Pillow's convolution resampler runs on the reduced image (or C) with the box as C floats: scale = (double)(x1 - x0) / W_t,
 *      centre = x0 + (j + 0.5) scale. An axis is resampled when its size changes or its box is not (0, size): Pillow's
 *      need_horizontal / need_vertical. The tall-image deviation of DESIGN §13 stays.
 *   3. The window selects output columns and rows of the two tables: every output pixel depends only on its own table row, so the
 *      cropped resize is exact.
 * b200jpg_batch_output_extent, out_bytes / out_offset and the descriptor rules of b200jpg_batch_decode_into(_ex) describe ww x wh.
 * The reconstruction covers only the part of C the tables (or the reduce box) read; the frame's status is its status without
 * the size. A batch in which some frame reduces issues one launch more than without the reduce.
 * boxes and windows NULL or all zero, and reducing_gap <= 0: exactly b200jpg_batch_create_draft. Otherwise, for the call,
 * tolerate_bad or not, B200JPG_ERR_INVALID_PARAMETER with the frame named in the message: a box or window on a frame without a
 * size; a box that is not finite, has a negative offset, leaves C or has x1 < x0 or y1 < y0; a window outside W_t x H_t or with
 * a zero side; a reduce box that is empty (Pillow raises there too); a reducing_gap that is NaN or in (0, 1). A frame whose
 * fx * fy reaches 2^24 is B200JPG_ERR_NOT_IMPLEMENTED for the call. The box and window of a frame that fails to parse are
 * ignored. */
B200JPG_API int b200jpg_batch_create_resample(b200jpg_ctx *ctx, const uint8_t *const *frames, const size_t *lens, int n, int tolerate_bad,
                                              unsigned flags, const b200jpg_size *drafts, const b200jpg_rect *rects, const b200jpg_size *sizes,
                                              const b200jpg_box *boxes, const b200jpg_rect *windows, int resample, double reducing_gap,
                                              b200jpg_batch **batch);
/* The flips of b200jpg_batch_create_flip, or-ed into one entry per frame. */
#define B200JPG_FLIP_H 1
#define B200JPG_FLIP_V 2
/* b200jpg_batch_create_resample with a flip per frame (DESIGN §21; no counterpart in the reference), torchvision's
 * RandomHorizontalFlip / RandomVerticalFlip and PIL's FLIP_LEFT_RIGHT / FLIP_TOP_BOTTOM. The flip is the last geometric step:
 * draft / downscale -> mode -> orientation -> crop -> resize -> window -> flip -> float map. Let O be what frame i is written as
 * without it ([h, w, C]); with flips[i] it is written as O[:, ::-1] (B200JPG_FLIP_H), O[::-1, :] (B200JPG_FLIP_V) or O[::-1, ::-1]
 * (both), for every destination kind; with B200JPG_FLAG_NO_UPSAMPLE every plane is flipped at its own extent. Rectangles, sizes,
 * boxes and windows keep their coordinates (those of the unflipped image). A flip changes no extent, out_bytes / out_offset,
 * status or b200jpg_batch_frame_orientation (the Exif value). A flipped frame without a size is planned as the frame of the
 * composed orientation, its rectangle mirrored, and joins that orientation's reconstruction group; a resized frame's resample
 * pass stores mirrored, with the launches of the unflipped batch. flips == NULL, or every entry 0: exactly
 * b200jpg_batch_create_resample. An entry with any other bit set is B200JPG_ERR_INVALID_PARAMETER for the call, tolerate_bad or not,
 * the frame named in the message. The flip of a frame that fails to parse is ignored. */
B200JPG_API int b200jpg_batch_create_flip(b200jpg_ctx *ctx, const uint8_t *const *frames, const size_t *lens, int n, int tolerate_bad,
                                          unsigned flags, const b200jpg_size *drafts, const b200jpg_rect *rects, const b200jpg_size *sizes,
                                          const b200jpg_box *boxes, const b200jpg_rect *windows, int resample, double reducing_gap,
                                          const uint8_t *flips, b200jpg_batch **batch);
/* Pillow's draft scale of one codestream for a requested width x height (host only): s = min(W / width, H / height) in integer
 * division over the codestream's own W x H (before any Exif orientation), and the largest k of 8, 4, 2, 1 with k <= s, or 1 when
 * none fits. Returns k, or the negative parse error of the codestream; a zero width or height is B200JPG_ERR_INVALID_PARAMETER. */
B200JPG_API int b200jpg_draft_scale(const uint8_t *data, size_t len, uint32_t width, uint32_t height);
/* The fixed-point tables b200jpg_batch_create_resize uses to resample one axis of in_size samples to out_size (tests only, host
 * only, no device): bounds[2 j] is the first source index and bounds[2 j + 1] the number of taps of output j, coeffs[j * ksize + t]
 * the int32 coefficient of tap t (zero behind the taps). *ksize receives the row length. The tables are written when bounds and
 * coeffs are both non-NULL: bounds needs 2 * out_size entries and coeffs `capacity` >= out_size * ksize entries, else the call
 * returns B200JPG_ERR_INVALID_PARAMETER. Also B200JPG_ERR_INVALID_PARAMETER: a zero size, an unknown filter or a NULL ksize.
 * For B200JPG_RESAMPLE_CV_LINEAR / _CV_AREA the tables are OpenCV's (DESIGN §20), of the horizontal axis, or of the vertical one
 * with B200JPG_CV_TABLE_VERTICAL or-ed into `resample`:
 *   - INTER_LINEAR, and INTER_AREA on an axis that upscales or with B200JPG_CV_TABLE_LINEAR (the other axis upscales): ksize = 2,
 *     bounds[2 j] and bounds[2 j + 1] the two source indices of output j (clamped to the axis), coeffs[2 j], coeffs[2 j + 1] their
 *     int16 weights (11 fractional bits);
 *   - INTER_AREA otherwise: bounds as for Pillow's filters (first source index, taps), coeffs[j * ksize + t] the bits of the float
 *     weight of tap t (computeResizeAreaTab). The batch sums blocks instead where both axes shrink by integer factors. */
#define B200JPG_CV_TABLE_VERTICAL 0x1000
#define B200JPG_CV_TABLE_LINEAR 0x2000
B200JPG_API int b200jpg_resample_coefficients(uint32_t in_size, uint32_t out_size, int resample, int32_t *bounds, int32_t *coeffs,
                                              uint64_t capacity, uint32_t *ksize);
/* b200jpg_resample_coefficients for the source box [in0, in1) of b200jpg_batch_create_resample, as Pillow's C resampler takes it in
 * floats (tests only, host only). Also B200JPG_ERR_INVALID_PARAMETER: a box that is not 0 <= in0 <= in1 <= in_size, and the
 * OpenCV filters, which take no box. */
B200JPG_API int b200jpg_resample_coefficients_box(uint32_t in_size, float in0, float in1, uint32_t out_size, int resample, int32_t *bounds,
                                                  int32_t *coeffs, uint64_t capacity, uint32_t *ksize);
/* The uncropped output size W_o x H_o of one codestream under `flags` (B200JPG_FLAG_DOWNSCALE_k, and width and height swapped for
 * the Exif orientations 5..8 with B200JPG_FLAG_EXIF_ORIENTATION; the frame size, B200JPG_FLAG_NO_UPSAMPLE or not): what the crop
 * rectangles of b200jpg_batch_create_crop are checked against. Returns B200JPG_OK or the error code b200jpg_parse returns for it
 * (B200JPG_ERR_INVALID_PARAMETER for a NULL width or height). Host only, no device. */
B200JPG_API int b200jpg_output_size(const uint8_t *data, size_t len, unsigned flags, uint32_t *width, uint32_t *height);
/* Waits for the work last enqueued for this batch (its buffers return to the context's pool for reuse by the
 * next batch; b200jpg_destroy frees the pool). The caller must have consumed `out_dev` before reusing it. */
B200JPG_API void b200jpg_batch_destroy(b200jpg_batch *batch);

B200JPG_API int b200jpg_batch_frame_info(const b200jpg_batch *batch, int i, b200jpg_frame_info *info);
/* Width and height of component c of frame i as the decode entry points write it: the frame size (reduced by
 * B200JPG_FLAG_DOWNSCALE_k), or the component's own size with B200JPG_FLAG_NO_UPSAMPLE. Returns B200JPG_OK, the frame's parse
 * status for a frame that failed (nothing written), or B200JPG_ERR_INVALID_PARAMETER. b200jpg_batch_frame_info keeps the
 * codestream's geometry. */
B200JPG_API int b200jpg_batch_output_extent(const b200jpg_batch *batch, int i, int c, uint32_t *width, uint32_t *height);
/* The number of components frame i is written with: its own, or 3 / 1 with B200JPG_FLAG_OUTPUT_RGB / B200JPG_FLAG_OUTPUT_L. The
 * frame's status for a frame that failed, B200JPG_ERR_INVALID_PARAMETER for a bad index. */
B200JPG_API int b200jpg_batch_output_components(const b200jpg_batch *batch, int i);
/* Frame i's Exif orientation 1..8, whether or not the batch applies it (B200JPG_FLAG_EXIF_ORIENTATION); the frame's status for a
 * frame that failed, B200JPG_ERR_INVALID_PARAMETER for a bad index. */
B200JPG_API int b200jpg_batch_frame_orientation(const b200jpg_batch *batch, int i);
/* Byte offset / size of frame i inside the batch output buffer; total size with i = -1. */
B200JPG_API uint64_t b200jpg_batch_out_offset(const b200jpg_batch *batch, int i);
B200JPG_API uint64_t b200jpg_batch_out_bytes(const b200jpg_batch *batch, int i);
/* Algorithmic-traffic accounting for the roofline (SURVEY.md 8d): ECS bytes and stored blocks of the batch. */
B200JPG_API uint64_t b200jpg_batch_ecs_bytes(const b200jpg_batch *batch);
B200JPG_API uint64_t b200jpg_batch_stored_blocks(const b200jpg_batch *batch);
B200JPG_API uint64_t b200jpg_batch_h2d_bytes(const b200jpg_batch *batch);

/* Replace the Huffman/quantisation table blob of this batch by an externally supplied device-independent
 * blob (multi-GPU: rank 0 exports, NCCL broadcasts, other ranks import). export returns the size. */
B200JPG_API uint64_t b200jpg_batch_export_tables(const b200jpg_batch *batch, uint8_t *dst, uint64_t capacity);
B200JPG_API int b200jpg_batch_import_tables(b200jpg_batch *batch, const uint8_t *src, uint64_t size);

/* H2D of the packed codestream bytes + descriptors on `stream` (a cudaStream_t, 0 = default). */
B200JPG_API int b200jpg_batch_upload(b200jpg_batch *batch, void *stream);

/* Re-runs only the device-side restart index that b200jpg_batch_upload builds behind its copy (EntropyParser::
 * ParseRestartMarker bookkeeping, codestream/entropyparser.cpp:117-136) -- idempotent; lets a caller time it. */
B200JPG_API int b200jpg_batch_reindex(b200jpg_batch *batch, void *stream);

/* The hot path: entropy decode kernel(s) then reconstruction kernel(s), asynchronous on `stream`.
 * `out_dev` is a DEVICE pointer to b200jpg_batch_out_bytes(batch,-1) bytes. */
B200JPG_API int b200jpg_batch_decode(b200jpg_batch *batch, uint8_t *out_dev, void *stream);
/* Where component c of a frame goes, the device-side ImageBitMap of interface/imagebitmap.hpp:104-109 (ibm_pData,
 * ibm_cBytesPerPixel, ibm_lBytesPerRow): the sample at (x, y) is written at
 *     data + x * bytes_per_pixel + y * bytes_per_row      (both strides signed: BGR order, padded rows, bottom-up images)
 * Samples are bytes for 8-bit frames, native-endian 16-bit for 12-bit frames (as in the packed output). */
typedef struct b200jpg_plane {
    void *data;
    int32_t bytes_per_pixel;
    int32_t pad;
    int64_t bytes_per_row;
} b200jpg_plane;

/* b200jpg_batch_decode with caller-described destinations, what the reference's BitMapHook hands out per component
 * (interface/bitmaphook.cpp, BitmapCtrl::RequestUserData control/bitmapctrl.cpp:142): planes[4*i + c] for frame i (the caller's frame index; JPEG XT residual
 * codestreams own no output), component c < ncomp.  Component geometry is what the batch was created with: width x height,
 * or ceil(width/subx[c]) x ceil(height/suby[c]) with B200JPG_FLAG_NO_UPSAMPLE, each reduced with B200JPG_FLAG_DOWNSCALE_k
 * (b200jpg_batch_output_extent).
 * For every frame the call writes exactly the samples b200jpg_batch_decode writes into that frame's slot (damaged frames
 * under tolerate_bad included), rearranged, and nothing else: bytes between pixels and between rows keep their contents.
 * A frame whose parse failed has no destination (its data may be NULL).  Overlap between components or frames is the
 * caller's responsibility, as in the reference.  Returns B200JPG_ERR_INVALID_PARAMETER and launches nothing when a live
 * frame has a NULL data, a pointer is not device (or managed) memory of the batch's device, |bytes_per_pixel| is below the
 * sample size, |bytes_per_row| < width * |bytes_per_pixel| for a component more than one row high, or a 16-bit destination
 * is not 2-byte aligned in data or in either stride.  `planes` may be reused as soon as the call returns; the call issues
 * as many kernel launches as b200jpg_batch_decode. */
B200JPG_API int b200jpg_batch_decode_into(b200jpg_batch *batch, const b200jpg_plane *planes, void *stream);
/* Float destinations: every sample v that b200jpg_batch_decode_into would write (0..255, or 0..4095 for 12-bit frames) is
 * written as
 *     y = fp32_round(fp32_round((float)v * scale[c]) + bias[c])      (two roundings, no fused multiply-add)
 * stored as float32, or rounded to nearest even into float16 (overflow -> inf, subnormals kept) or bfloat16. c is the output
 * component: R, G, B after the colour transformation, else the frame's component / plane index. One map per call, uniform
 * over the batch's frames. */
#define B200JPG_SAMPLE_F32 1
#define B200JPG_SAMPLE_F16 2
#define B200JPG_SAMPLE_BF16 3
typedef struct b200jpg_convert {
    int32_t type; /* B200JPG_SAMPLE_* */
    float scale[B200JPG_MAX_COMPONENTS], bias[B200JPG_MAX_COMPONENTS];
} b200jpg_convert;
/* b200jpg_batch_decode_into with the samples converted by `convert` (NULL: exactly b200jpg_batch_decode_into). The
 * descriptor rules are those above with the element size (4 bytes for float32, 2 for float16 / bfloat16) in place of the
 * sample size: |bytes_per_pixel| >= element size, no overlapping rows, data and both strides aligned to the element size.
 * Also B200JPG_ERR_INVALID_PARAMETER, with nothing launched: an unknown type, or a non-finite scale or bias of a component
 * that a live frame of the batch has. The call writes the same positions as b200jpg_batch_decode_into and issues as many
 * kernel launches. */
B200JPG_API int b200jpg_batch_decode_into_ex(b200jpg_batch *batch, const b200jpg_plane *planes, const b200jpg_convert *convert,
                                             void *stream);
/* Per-component sample tables (DESIGN §22; host memory): every 8-bit sample v of output component c that
 * b200jpg_batch_decode_into would write is written as table[c][v], stored as float32, or rounded to nearest even into float16
 * (overflow -> inf, subnormals kept) or bfloat16, as b200jpg_convert's results are. A table holds any per-sample map exactly:
 * torchvision's ToTensor() + Normalize(mean, std) (three roundings, two divisions), gamma or sRGB curves, dequantisation. */
typedef struct b200jpg_convert_table {
    int32_t type; /* B200JPG_SAMPLE_* */
    float table[B200JPG_MAX_COMPONENTS][256];
} b200jpg_convert_table;
/* b200jpg_batch_decode_into_ex with the map replaced by `table`: the same descriptor rules, positions written and kernel launches
 * (the tables ride the call's one descriptor copy). B200JPG_ERR_INVALID_PARAMETER, with nothing launched: a NULL table or an
 * unknown type; B200JPG_ERR_NOT_IMPLEMENTED: a batch with a live 12-bit frame. */
B200JPG_API int b200jpg_batch_decode_into_table(b200jpg_batch *batch, const b200jpg_plane *planes, const b200jpg_convert_table *table,
                                                void *stream);
/* Only one of the two stages (profiling / roofline measurements / parity of the intermediate). */
B200JPG_API int b200jpg_batch_decode_entropy(b200jpg_batch *batch, void *stream);
B200JPG_API int b200jpg_batch_reconstruct(b200jpg_batch *batch, uint8_t *out_dev, void *stream);

/* After the stream has been synchronised: per-frame status (0 or a negative error code). Performs a small
 * D2H copy of the error words on first use. */
B200JPG_API int b200jpg_batch_frame_status(b200jpg_batch *batch, int i);

/* Debug / parity access: copies the dequantised coefficient plane of component c of frame i to the host
 * as int16 [blocks_h][blocks_w][64] in raster order inside the block. */
B200JPG_API int b200jpg_batch_read_coefficients(b200jpg_batch *batch, int i, int c, int16_t *dst, uint64_t capacity_elems);

/* Number of kernel launches the last b200jpg_batch_decode* call issued. */
B200JPG_API int b200jpg_batch_last_launch_count(const b200jpg_batch *batch);
/* CUDA-event timing of the two stages of the last decode call when timing is enabled (ms); timing makes
 * the call record events on `stream`, it does not synchronise. Read after synchronising. */
B200JPG_API void b200jpg_batch_enable_timing(b200jpg_batch *batch, int on);
B200JPG_API int b200jpg_batch_last_timing(b200jpg_batch *batch, float *entropy_ms, float *reconstruct_ms);
/* Share of entropy_ms spent in the unstuffing pre-pass (stage a0), ms; negative when not available. */
B200JPG_API float b200jpg_batch_last_unstuff_ms(b200jpg_batch *batch);

/* Measured int32 issue rate of the device in Gop/s (integer multiply-add counted as 2 ops, SURVEY.md 8d):
 * multiply-add only, add/logic only, and a 1:1 mix. Denominator of the reconstruction kernel's roofline. */
B200JPG_API int b200jpg_microbench_int32(int device, float *imad_gops, float *alu_gops, float *mix_gops);

/* Self-test of the host logic behind restart-less scans (tests only, no device): replays the synchronisation rounds of the
 * device kernel for scan 0 of one codestream on the host and checks the resulting work items against a front-to-back walk.
 * Returns B200JPG_OK, a parser error, or -1..-4 for an inconsistent partition. */
B200JPG_API int b200jpg_selftest_restartless(const uint8_t *data, size_t len, uint32_t *rounds, uint32_t *n_segments);
/* The work items of the same host replay (tests only, no device), seven int32 per item: start bit in the unstuffed scan, first
 * block, block count and the DC predictors of the four scan components. *n_items receives the count; with fewer than that in
 * `cap` nothing is written and the call returns B200JPG_ERR_INVALID_PARAMETER. */
B200JPG_API int b200jpg_selftest_restartless_items(const uint8_t *data, size_t len, int32_t *items, uint32_t cap, uint32_t *n_items,
                                                   uint32_t *rounds);
/* Host-only self-test of the decoder-table cache of b200jpg_batch_create (frames of one source share their tables; the tables of a
 * scan are built once per distinct set of Huffman specifications, quantisation tables and scan parameters): every scan of the
 * given codestreams through the cache, twice, against a fresh HuffmanTemplate::BuildDecoder-equivalent build
 * (coding/huffmantemplate.cpp:802-874).  Returns the number of scans compared, or a negative value on a mismatch. */
B200JPG_API int b200jpg_selftest_table_cache(const uint8_t *const *frames, const size_t *lens, int n);

/* One-call convenience used by the C++ JPEG shim: host codestreams in, HOST pixels out (upload, decode,
 * download, synchronise).  `out_host` receives b200jpg_batch_out_bytes(batch,-1) bytes. */
B200JPG_API int b200jpg_decode_to_host(b200jpg_ctx *ctx, const uint8_t *const *frames, const size_t *lens, int n, uint8_t *out_host,
                           uint64_t out_capacity);
B200JPG_API int b200jpg_decode_to_host_ex(b200jpg_ctx *ctx, const uint8_t *const *frames, const size_t *lens, int n, uint8_t *out_host,
                              uint64_t out_capacity, unsigned flags);

/* The same, but the pixels STAY ON THE DEVICE (consumers that work on the GPU skip the PCIe copy of 24.9 MB per 4K frame, SURVEY 5):
 * *out_dev receives a device buffer (frame i at the 256-byte aligned running offset, frame 0 at 0; *out_bytes its size), to be
 * released with b200jpg_device_free.  b200jpg_device_copy_rect copies a rectangle of rows between two device bitmaps (for clients
 * that keep an interleaved device canvas of their own; JPEG::DisplayRectangle with JPGTAG_B200_DEVICE_BITMAPS copies into the
 * client's per-component bitmaps with a kernel of its own). */
B200JPG_API int b200jpg_decode_to_device_ex(b200jpg_ctx *ctx, const uint8_t *const *frames, const size_t *lens, int n, unsigned flags,
                                uint8_t **out_dev, uint64_t *out_bytes);
B200JPG_API void b200jpg_device_free(b200jpg_ctx *ctx, uint8_t *p);
B200JPG_API int b200jpg_device_copy_rect(b200jpg_ctx *ctx, uint8_t *dst_dev, int64_t dst_pitch, const uint8_t *src_dev, int64_t src_pitch,
                             uint64_t width_bytes, uint64_t rows);

#ifdef __cplusplus
}
#endif
#endif
