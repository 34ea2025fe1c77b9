// internal.hpp -- shared declarations of the GPU baseline-JPEG decode path (host parser <-> CUDA stages).
//
// Data layout in HBM (one "batch" = n codestreams decoded by the same launches):
//   bytes      : the codestreams, each copied whole at a 16-byte aligned offset and followed by FF D9 + zero
//                padding, so a bit reader that runs off a damaged segment always meets a marker.
//   clean      : the entropy coded segments with byte stuffing removed, one 16-byte aligned run per restart
//                interval, stored as big-endian 32-bit words and followed by >= 32 zero bytes (stage a0 output).
//   coef       : int16, one 128-byte block per 8x8 DCT block, DEQUANTISED (coefficient * delta, the << 4
//                preshift of dct/idct.cpp:105 is applied by the reconstruction kernels), raster order inside
//                the block; per component a plane [blocks_h][blocks_w] over the MCU-padded grid.
//   samples    : int32, IDCT output (4 fractional bits, level shifted) of the SUBSAMPLED components only,
//                plane [8*blocks_h][8*blocks_w] -- the role of the reference's upsampler line buffers
//                (upsampling/upsamplerbase.cpp:300-327), whole-frame instead of a sliding window.
//   out        : interleaved 8-bit pixels, caller-provided.
#pragma once
#include <cstddef>
#include <cstdint>
#include <string>
#include <vector>

#include "b200jpg.h"

namespace b200jpg {

// ---- host-side parse results -------------------------------------------------------------------------
struct HuffSpec {  // DHT payload, coding/huffmantemplate.cpp:878-904
    bool defined = false;
    uint8_t bits[16] = {0};
    uint8_t vals[256] = {0};
    int nvals = 0;
};

struct ScanInfo {  // one SOS + its entropy coded segment
    int ns = 0;
    int comp[4] = {0, 0, 0, 0};  // frame component index, SOS order
    int td[4] = {0, 0, 0, 0}, ta[4] = {0, 0, 0, 0};
    int lowbit = 0;              // point transform Al
    // progressive frames (SOF2): spectral selection Ss..Se and the bit position Ah of the previous pass of this band
    // (0: first pass); sequential scans have 0, 63, 0
    bool progressive = false;
    int ss = 0, se = 63, ah = 0;
    uint32_t dri = 0;            // MCUs per restart interval, 0 = none
    size_t ecs_off = 0, ecs_end = 0;
    uint32_t mcu_cols = 0, mcu_rows = 0;
    // byte offset (within the codestream) of the first ECS byte of every restart interval;
    // SIZE_MAX marks an interval the stream does not contain (zero-filled like an invalid segment,
    // codestream/sequentialscan.cpp:415-419)
    std::vector<size_t> interval_off;
    std::vector<size_t> interval_end;  // offset of the marker (or end of data) that terminates the interval
    // true: the host did not walk the entropy coded segment; ecs_end is the offset of the closing EOI and the restart
    // index above is a placeholder that restart_index_kernel fills in on the device (SURVEY 8f1)
    bool device_index = false;
    // the data ends inside this scan's last restart interval (no marker behind it): the decoder reads zero bits there and
    // must not report the overrun (the reference does not, io/bitstream.cpp:103-105)
    bool eof_tail = false;
    // a sequential scan without restart markers that is long enough to be worth cutting up: decoded through synchronisation
    // points (specsync.hpp) instead of by a single lane
    bool spec = false;
    HuffSpec dc[4], ac[4];       // tables in effect at this SOS
    uint16_t quant[4][64];       // zig-zag order; slot tq of a scan component holds that component's ParsedFrame::comp_quant
    bool quant_defined[4] = {false, false, false, false};
};

// JPEG XT (ISO/IEC 18477) residual layer of a frame, SURVEY 8f3: what the APP11 boxes in front of the first scan say
// (boxes/box.cpp:95-205, boxes/mergingspecbox.cpp, boxes/outputconversionbox.cpp:92-127, boxes/colortrafobox.cpp:55-78).
// Covered: the 8-bit integer profile the reference encoder writes with `-r -q -Q` -- an ordinary DCT codestream in the RESI
// box, merged per pixel (YCbCrTrafo::YCbCr2RGB colortrafo/ycbcrtrafo.cpp:747-880) with default (identity) tables, clamped
// output.  Anything else that is present makes the frame NOT_IMPLEMENTED; it is never decoded as if the boxes were absent.
struct XtLayer {
    bool present = false;      // a merging specification and a residual codestream were found and are covered
    bool l_ycbcr = false;      // base image: YCbCr -> RGB before the merge
    bool r_ycbcr = false;      // residual image: YCbCr -> RGB before the merge
    std::vector<uint8_t> resi;  // the residual codestream, reassembled from its APP11 pieces
};

struct ParsedFrame {
    b200jpg_frame_info info{};
    std::vector<ScanInfo> scans;
    XtLayer xt;
    // Exif orientation (tag 0x0112 of IFD0 in the first APP1 "Exif\0\0" segment in front of the first scan), 1..8; 1 when there
    // is none or it is malformed. Applied only with B200JPG_FLAG_EXIF_ORIENTATION; never changes the parse status
    int orientation = 1;
    // the transform byte (payload[11]) of the last APP14 segment in front of the first scan whose payload has at least 12 bytes and
    // starts with "Adobe" (libjpeg's examine_app14), -1 when there is none. Only the colour space of four-component frames follows
    // it (frame_colorspace); three-component frames keep the reference's rule (b200jpg_frame_info::ycbcr)
    int adobe_transform = -1;
    // the quantiser of each frame component (zig-zag order), latched at the first scan that contains the component: the
    // reference builds a component's inverse DCT once, at that scan (BlockBuffer::ResetToStartOfScan control/blockbuffer.cpp:
    // 185-197, IDCT::DefineQuant dct/idct.cpp:98-108), so a DQT that redefines the slot later does not reach it. Every
    // consumer reads this: the scans' table sets (ScanInfo::quant of the scan's components), the fused DC kernel and the
    // scan-by-scan dequantisation
    uint16_t comp_quant[4][64];
};

// B200JPG_COLORSPACE_* of a parsed frame: grey, YCbCr / RGB by b200jpg_frame_info::ycbcr, CMYK / YCCK for an 8-bit four-component
// frame with an Adobe segment (transform 0: CMYK, any other value: YCCK, libjpeg's default_decompress_parms), else unknown
int frame_colorspace(const ParsedFrame &pf);

// The orientation an APP1 payload (the bytes behind the length field) gives: 0 when it is not an Exif segment, else 1..8
// (1 for anything malformed)
int exif_orientation_of(const uint8_t *s, size_t rem);

// Returns 0 or a negative reference error code; `err` receives a message. With `device_index` a scan that carries all
// components of the frame and uses restart markers is not walked on the host (ScanInfo::device_index).
int parse_codestream(const uint8_t *data, size_t len, ParsedFrame &out, std::string &err, bool device_index = false);

// Restart bookkeeping with the reference's resynchronisation (codestream/entropyparser.cpp:117-199) over the marker
// sequence of one entropy coded segment; off / end are sized to the number of restart intervals (parse.cpp).
int resolve_restart_sequence(const std::vector<size_t> &rst_at, const std::vector<uint8_t> &rst_id, size_t ecs_off, size_t ecs_end,
                             bool ended_by_eof, std::vector<size_t> &off, std::vector<size_t> &end);

extern const uint8_t kZigZagToRaster[64];  // dct/dct.cpp:57-73

// ---- table sets: what the entropy kernel needs besides the bytes ------------------------------------
// Serialised, device independent (this blob is what rank 0 broadcasts over NCCL):
//   uint32 magic, uint32 total_bytes, uint32 lut_words, uint32 flags
//   uint16 lut_off[8]        word offset of the first-level LUT of DC0..3, AC0..3 (0xFFFF = undefined)
//   uint32 qz[4][160][2]     per quantisation table, index = zig-zag position k: {delta << lowbit, byte offset of the
//                            raster position inside a block}; entries 64..95 multiply by 2^16 (a coefficient whose run
//                            leaves the block overflows the int16 store: out-of-sync error; a ZRL that leaves it carries
//                            amplitude 0 and just ends the block), entries 96..159 are where "the block ends" symbols
//                            land (no error); both kinds point at the staging block's pad slot
//   uint32 lut[lut_words]    per table: 2^kLutL1Bits first-level entries, then 2^(16-kLutL1Bits) per second-level table
// LUT entry: [4:0] s = value bits that follow the code, [9:5] code length (0: pointer to second-level table
// [17:10], all other fields 0; 31: unused code, coding/huffmandecoder.hpp:87), [25:19] step of the zig-zag index
// (AC: run + 1, ZRL 16, EOB and error entries kQzBlockEnds), [30:26] total = length + s, [31] decoding this entry is
// an error (unused code, DC category > 15, AC symbol that baseline does not define).
constexpr uint32_t kTableMagic = 0x4a54424du;  // "MBTJ"
constexpr int kLutL1Bits = 11;  // 2 KB entries per table; at q75 fewer than 0.4 % of the AC codes are longer
constexpr int kQzEntries = 160;    // per quantisation table, see above
constexpr int kQzBlockEnds = 96;   // zig-zag step of symbols that end the block: lands in the entries 96..159
constexpr int kTableHeaderBytes = 16 + 16 + 4 * kQzEntries * 2 * 4;

struct TableSet {
    std::vector<uint8_t> blob;
    uint32_t lut_words() const;
};

// Builds the blob for one scan (two-level decoder tables, coding/huffmantemplate.cpp:802-874).
int build_table_set(const ScanInfo &scan, TableSet &out, std::string &err);

// ---- device-side descriptors -------------------------------------------------------------------------
struct ClassScan {        // one scan of one frame inside a scan class
    uint64_t coef_base[4];  // element (int16) offset of the plane of scan component c
    uint32_t frame;         // index into the batch
    uint32_t pad;
};

// One scan whose restart index is built on the device. Offsets are bytes inside the batch's input buffer; the three
// arrays are this scan's slices of its class's interval arrays.
struct IndexScan {
    uint64_t ecs_off, ecs_end;                 // first entropy coded byte, offset of the closing EOI
    uint64_t off_arr, end_arr, clean_arr;      // uint64[n_intervals] each
    uint64_t clean_base;                       // start of the scan's region in the unstuffed buffer (16-byte aligned)
    uint32_t n_intervals, frame;
};
constexpr uint32_t kCleanSlackPerInterval = 80;  // device-indexed scans: clean_off[k] = base + (off[k] - ecs_off) + 80 k, 16-aligned
int launch_restart_index(const IndexScan *scans_dev, uint32_t n_scans, uint8_t *input_dev, uint32_t *index_status, void *stream);

// bit 63 of an interval_end entry / bit 31 of an interval_len entry: the data (not a marker) ends this interval -- the
// decoder reads zero bits behind it like the reference's bit reader at EOF and does not report the overrun
constexpr uint64_t kIntervalEofFlag = 1ull << 63;
constexpr uint32_t kIntervalLenEofFlag = 1u << 31;
// bit 30 of an interval_len entry: the stream does not contain this interval (its MCUs stay cleared). An interval that is
// present but EMPTY (two restart markers back to back) is decoded -- from zero bits, like the reference does
constexpr uint32_t kIntervalLenAbsent = 1u << 30;
constexpr uint32_t kIntervalLenMask = (1u << 30) - 1u;

struct SpecSegment;
struct SpecLog;

struct ScanClassParams {  // uniform over a launch of the entropy kernel
    int ns;
    int mw[4], mh[4];       // blocks per MCU of scan component c (1,1 for single component scans)
    int bw[4];              // plane pitch in blocks of scan component c
    int dc_slot[4], ac_slot[4], q_slot[4];
    uint32_t mcu_cols, total_mcus, dri /* MCUs per interval, >= 1 */, intervals_per_scan;
    uint32_t n_scans;       // scans in this class
    uint32_t lut_words;
    // progressive scans (SOF2): handled by progressive_scan_kernel instead of entropy_decode_kernel
    int progressive, ss, se, ah, al;
    int ordinal;            // position of the scan inside its frame: progressive classes are launched in this order
    // restart-less sequential scans decoded through synchronisation points (specsync.hpp): the scan is ONE interval to the
    // unstuffing kernel and segs_per_scan work items (SpecSegment) to the decoder
    int indexed;
    uint32_t segs_per_scan;
};

// One progressive frame for the dequantisation pass that follows its last scan: the progressive kernels keep
// quantised levels in the coefficient store, stage b expects dequantised coefficients.
struct ProgFrame {
    uint64_t coef_base[4];   // int16 element offsets of the component planes
    uint32_t n_blocks[4];    // blocks per plane (MCU-padded grid), 0 = component absent
    uint16_t q_raster[4][64];  // quantiser of the component in raster order
    uint32_t frame, pad;
};

// Component-fused progressive decoding (progfused_sm100.cu): one launch runs a restart interval through ALL scans of a group
// -- the interleaved DC scans of a frame, or the AC scans of one component -- in file order.
constexpr int kPfMaxScans = 6;
struct PfScan {                    // one scan of the group, uniform over the launch
    const uint8_t *tables;         // device copy of the scan's table-set blob
    const uint64_t *clean_off;     // [n_frames * intervals] offsets of the unstuffed intervals of this scan
    const uint32_t *interval_len;  // [..] unstuffed lengths (flags: kIntervalLenAbsent / kIntervalLenEofFlag)
    int ss, se, ah, al;
    int dc_slot[4], ac_slot, q_slot;
    uint32_t lut_words;
    int lut_share;                 // AC kernel: the first scan of the launch whose decoder tables are the same words (itself if none)
};
struct PfLaunch {
    int n_scans;
    PfScan scan[kPfMaxScans];
    int ns;                        // components in the group's scans (DC group: all of the frame; AC group: 1)
    int mw[4], mh[4], bw[4];       // blocks per MCU and plane pitch of scan component c
    uint32_t ac_cols[4], ac_rows[4];  // DC group: the block grid the component's own (single-component) scans cover
    uint16_t dc_quant[4];          // quantiser of coefficient 0 of scan component c
    uint32_t mcu_cols, total_mcus, dri, intervals, n_frames;
    const ClassScan *frames;       // [n_frames] coefficient plane of every scan component + frame index
    const uint8_t *clean;
    int16_t *coef;
    int16_t *dcplane;              // one quantised DC level per block, indexed like the coefficient store / 64
    uint32_t *frame_status;
};
int launch_pf_dc(const PfLaunch &L, void *stream);
int launch_pf_ac(const PfLaunch &L, void *stream);

struct FrameRecon {       // per frame, for the reconstruction kernels
    uint64_t coef_base[4];    // int16 element offsets
    uint64_t sample_base[4];  // element offsets into the sample planes (subsampled components only)
    uint64_t out_base;        // byte offset into the output buffer
    uint32_t width, height;
    uint32_t bw[4], bh[4];
    uint32_t ncomp, ycbcr, subx, suby;  // subx/suby of the subsampled (chroma) components
    uint32_t cw, ch;                    // true subsampled size ceil(W/subx), ceil(H/suby)
    uint32_t status_idx, precision;     // sample precision of the frame (8, or 12: generic reconstruction, 16-bit samples out)
    uint8_t csx[4], csy[4];             // generic reconstruction: subsampling factors of every component (1..4)
    // JPEG XT (generic reconstruction): bit 0 = merge with the residual image whose int32 sample planes start at
    // res_sample_base (block grid width res_bw, factors res_csx / res_csy), bit 1 / 2 = YCbCr -> RGB on the base / residual side.
    // ycck (groups of OutMode::CmykRgb / CmykLuma): 1 = the frame is YCCK, its first three samples go through YCC -> RGB first
    uint32_t xt, ycck;
    uint64_t res_sample_base[4];
    uint32_t res_bw[4];
    uint8_t res_csx[4], res_csy[4];
    // downscaled frames (ReconPath::Scaled / Scaled420): the coefficient block grid; bw / bh are then the grid of the reduced
    // sample planes, ceil(coef_bw / k) x ceil(coef_bh / k), and width / height the reduced frame
    uint32_t coef_bw[4], coef_bh[4];
    // cropped frames (groups launched with the clip kinds): the CTA at grid position (bx, by) runs tile (tx0 + bx, ty0 + by) of
    // the path's tile grid (recon_tile), and a sample (x, y) is stored only inside [clip_x0, clip_x1) x [clip_y0, clip_y1), in the
    // decoded coordinates of width x height. ReconPath::Tiled: b1 computes only chroma blocks [cb_x0, cb_x1) x [cb_y0, cb_y1)
    uint32_t tx0, ty0;
    uint32_t clip_x0, clip_y0, clip_x1, clip_y1;
    uint32_t cb_x0, cb_y0, cb_x1, cb_y1;
    // drafted frames (Turbo / TurboGeneric groups of ReconLaunch::downscale > 1, DESIGN §17): width / height are the reduced frame, bw / bh =
    // coef_bw / coef_bh the coefficient grid, and block (bx, by) of component c leaves the IDCT as idct[c] x idct[c] samples (8, 4,
    // 2 or 1) of a plane with row pitch idct[c] bw[c]; csx / csy are then the upsampling ratios after that IDCT, and fancy = 0 (1/8)
    // replicates every ratio
    uint8_t idct[4];
    uint32_t fancy;
};

// The tiles of the reconstruction kernels, in luma blocks (8 x 8 samples of the decoded frame): reconstruct_kernel (b2) runs 32 x
// kThreadsB / 32 blocks per CTA, reconstruct420_kernel and reconstruct420_scaled_kernel 32 x kRows420, generic_reconstruct_kernel
// kGenericTileBlocks x 1
constexpr int kThreadsB = 128;
#ifndef B200JPG_R420_ROWS
#define B200JPG_R420_ROWS 4
#endif
constexpr int kRows420 = B200JPG_R420_ROWS;
constexpr int kGenericTileBlocks = 64;
struct ReconTile {
    uint32_t bw, bh;
};

// kernel launchers (huffman_sm100.cu, recon_sm100.cu). All asynchronous on `stream`.
struct EntropyLaunch {
    ScanClassParams p;
    const uint8_t *bytes;           // packed codestreams
    const uint64_t *interval_off;   // [n_scans * intervals_per_scan] first ECS byte, ~0ull = absent
    const uint64_t *interval_end;   // [..] offset of the marker that ends the interval
    const uint64_t *clean_off;      // [..] 16-byte aligned offset of the interval's unstuffed bytes in `clean`
    uint8_t *clean;                 // unstuffed, big-endian-word entropy coded data (written by a0, read by a1)
    uint32_t *interval_len;         // [..] unstuffed length in bytes (written by a0)
    const ClassScan *scans;         // [n_scans]
    const uint8_t *tables;          // device copy of the table-set blob
    int16_t *coef;
    uint32_t *frame_status;         // [n_frames]
    // sequential scans: {count, interval indices ...} of the intervals whose decoder read past the marker that ends them;
    // overrun_verdict_kernel replays exactly those with the reference's bit-reader bookkeeping to decide whether the
    // reference would have thrown (io/bitstream.hpp:168-208, bitstream.cpp:56-118)
    uint32_t *overrun_list;
    // indexed classes (p.indexed): work items written by spec_sync_kernel and its scratch, [n_scans * segs_per_scan] each
    struct SpecSegment *spec_segments;
    unsigned long long *spec_exits, *spec_entries;
    uint32_t *spec_counts;
    int32_t *spec_dc_sums;  // [.. * 4]
    struct SpecLog *spec_logs;
};
int launch_unstuff(const EntropyLaunch &l, void *stream);
int launch_entropy(const EntropyLaunch &l, void *stream);
int launch_overrun_verdict(const EntropyLaunch &l, void *stream);
int launch_spec_sync(const EntropyLaunch &l, void *stream);  // specsync_sm100.cu
// progressive_sm100.cu: one scan class of progressive frames; quantised levels -> dequantised coefficients afterwards
int launch_progressive_scan(const EntropyLaunch &l, void *stream);
int launch_progressive_dequant(const ProgFrame *frames_dev, uint32_t n_frames, uint32_t max_blocks, int16_t *coef, uint32_t *frame_status,
                               void *stream);

// How a frame goes from coefficients to pixels (abi.cpp: recon_path). Tiled: b1 planes of components 1.. + b2 (grey, 4:4:4,
// 4:2:2, 4:4:0); Fused420: reconstruct420_kernel, no planes; Generic: int32 planes of every component + the generic kernels
// Scaled (B200JPG_FLAG_DOWNSCALE_*): idct_scaled_planes_kernel into int32 planes laid out as the IDCT output of the reduced frame,
// then the generic kernels on a FrameRecon of the reduced width and height; Scaled420 (downscaled 8-bit 4:2:0 frames with
// upsampling): reconstruct420_scaled_kernel, no planes. B200JPG_FLAG_LIBJPEG_TURBO (DESIGN §16, turbo_sm90.cu): Turbo (grey, and
// three components with full-resolution component 0 and chroma factors 1 or 2, wider than 2 chroma samples when halved
// horizontally): turbo_idct_kernel into uint8 planes of components 1.., then turbo_reconstruct_kernel; TurboGeneric (every other
// such frame): uint8 planes of every reconstructed component, then turbo_generic_kernel. Frames drafted to 1/2, 1/4 or 1/8 (DESIGN
// §17) take the same two paths, decided on the ratios after their reduced IDCTs, through the _draft_ kernels
enum class ReconPath : int { Tiled, Fused420, Generic, Scaled, Scaled420, TurboGeneric, Turbo };
// B200JPG_FLAG_OUTPUT_RGB / _L (DESIGN §14): what a reconstruction group writes besides its components as they are. Luma: the generic
// kernels reduce three clamped components to L = (19595 R + 38470 G + 7471 B + 32768) >> 16 and store one; Replicate: a grey frame's
// sample is stored to three components. (An L frame of a YCbCr codestream is planned as a grey frame over its component 0: Coded.)
// CmykRgb / CmykLuma (DESIGN §15): the generic kernels turn four clamped samples of a CMYK or YCCK frame (FrameRecon::ycck) into
// Pillow's convert("RGB") and store three, or into its convert("L") and store one.
enum class OutMode : int { Coded, Luma, Replicate, CmykRgb, CmykLuma };
inline ReconTile recon_tile(ReconPath p) {
    if (p == ReconPath::Fused420 || p == ReconPath::Scaled420) return {32, (uint32_t)kRows420};
    if (p == ReconPath::Tiled || p == ReconPath::Turbo) return {32, (uint32_t)kThreadsB / 32};
    return {(uint32_t)kGenericTileBlocks, 1};
}
struct ReconLaunch {
    const FrameRecon *frames;  // device
    uint32_t n_frames;
    uint32_t max_bw0, max_bh0;     // largest luma block grid in the group
    uint32_t max_bwc, max_bhc;     // largest chroma block grid in the group
    uint32_t ncomp, subx, suby;    // uniform over the group
    ReconPath path;                // uniform over the group
    OutMode mode;                  // uniform over the group; not Coded only with described destinations (never kStoreCanvas)
    bool planes_out;               // B200JPG_FLAG_NO_UPSAMPLE: the components leave as planes at their own resolution
    int generic_phase;             // generic groups: 0 = IDCT then reconstruction, 1 = IDCT only, 2 = reconstruction only
    int downscale;                 // the group's factor k: B200JPG_FLAG_DOWNSCALE_k of Scaled groups, the draft of TurboGeneric groups
    const int16_t *coef;
    int16_t *samples16;            // chroma sample planes every frame goes through
    int32_t *samples32;            // the same planes for the exact pass over frames flagged `narrow`
    uint8_t *planes8;              // TurboGeneric groups: the uint8 planes (FrameRecon::sample_base are byte offsets into them)
    uint32_t *narrow_flags;        // [frames in batch], zeroed per decode: a chroma sample does not fit int16
    uint32_t *wide_flags;          // [frames in batch], zeroed per decode: a chroma sample leaves the 32-bit colour range
    uint32_t *narrow_list;         // [1 + frames in group] scratch: {count, group-local indices of the flagged frames}
    uint8_t *out;
    // b200jpg_batch_decode_into: where every component goes, [4 * frames in batch] indexed 4 * status_idx + c (device);
    // null: the packed slots of `out`
    const b200jpg_plane *planes;
    bool planar;                   // every plane of the group's frames has bytes_per_pixel == sample size (element size with `convert`)
    bool runs;                     // a group of Exif-oriented frames that is not planar, or of cropped frames: kStoreRuns / kStoreRunsF
    bool clip;                     // a group of cropped frames: the kinds with kStoreClip, grid over the tiles the crops cover
    // b200jpg_batch_decode_into_ex: the samples leave as float32 / float16 / bfloat16 through this map (host memory, passed to
    // the kernels by value); null: as integers
    const b200jpg_convert *convert;
    // b200jpg_batch_decode_into_table: with `convert` (its type), every sample v of output component c leaves as table[256 c + v]
    // (device); null: through the map
    const float *table;
};

// How the reconstruction kernels store a block (the destination kind of the launch, chosen per group from the descriptors):
// kStoreCanvas: the packed slot of `out` (b200jpg_batch_decode); kStorePlanar: one plane per component, samples adjacent;
// kStoreStrided: any signed pixel and row stride, one store per sample. kStorePlanarF / kStoreStridedF: the same layouts with
// float elements, every clamped integer sample v converted to fp32_round(fp32_round(v * scale[c]) + bias[c]) and rounded to
// the element type (B200JPG_SAMPLE_*, a launch-uniform switch inside the kind).
// kStoreRuns / kStoreRunsF (groups of Exif-oriented frames on the tiled 8-bit paths): the block is staged in the kernel's luma tile
// and leaves as runs of eight contiguous samples along x (mirrored rows) or along y (transposed), in either direction, a packed
// interleaved slot as 24-byte runs of pixels; whatever has no contiguous axis, one store per sample.
// kStoreClip, or-ed into kStoreRuns / kStoreRunsF / kStoreStrided / kStoreStridedF (groups of cropped frames): the CTAs run the tiles
// from FrameRecon::tx0 / ty0 on and store only inside the frame's clip rectangle; kBaseKind strips it.
// kStoreTable, or-ed into the float kinds (b200jpg_batch_decode_into_table): every sample leaves through FloatDst::table in place of
// the map. A bit of its own, so that the lookup is compiled out of the affine instances: in the 4:2:0 kernels it costs registers.
enum StoreKind : int { kStoreCanvas = 0, kStorePlanar = 1, kStoreStrided = 2, kStorePlanarF = 3, kStoreStridedF = 4, kStoreRuns = 5, kStoreRunsF = 6, kStoreClip = 8,
                       kStoreTable = 16 };
template <int k>
constexpr int kBaseKind = k & ~(kStoreClip | kStoreTable);
template <int k>
constexpr bool kClipKind = (k & kStoreClip) != 0;
template <int k>
constexpr bool kTableKind = (k & kStoreTable) != 0;
template <int k>
constexpr bool kFloatKind = kBaseKind<k> == kStorePlanarF || kBaseKind<k> == kStoreStridedF || kBaseKind<k> == kStoreRunsF;

// the destination argument of the float kinds: the descriptors plus the map, both in the kernel's parameter bank, and the
// per-component sample tables of b200jpg_batch_decode_into_table (device, 256 floats per component; null: the map), a
// launch-uniform switch like the element type
struct FloatDst {
    const b200jpg_plane *planes;
    int32_t type;
    float scale[B200JPG_MAX_COMPONENTS], bias[B200JPG_MAX_COMPONENTS];
    const float *table;
};
int launch_recon(const ReconLaunch &l, void *stream, int *launches);
// turbo_sm90.cu: a Turbo or TurboGeneric group, every frame cropped (ReconLaunch::clip), K = kStoreStrided or kStoreStridedF with
// kStoreClip, the latter also with kStoreTable
template <int K>
int launch_turbo(const ReconLaunch &l, void *stream, int *launches);

// ---- resize (b200jpg_batch_create_resize, DESIGN §13; boxes, reduce and windows of b200jpg_batch_create_resample, DESIGN §19),
// resample_sm100.cu. The reconstruction writes C, the frame's cropped output (the part of it the resize reads), as an interleaved
// uint8 bitmap into the batch's scratch; reduce_kernel reduces it to R behind it in the scratch where the frame reduces;
// resample_h_kernel runs the horizontal pass over the rows of the source (C or R) the vertical table touches into the
// intermediate, resample_v_kernel the vertical pass into the caller's destinations.
// The fixed-point tables of one axis of in_size samples for out_size outputs: bounds [out_size][2] int32 (first source index, taps),
// coefficients [out_size][ksize] int32 (zero behind the taps), PIL's convolution resampler; computed without floating-point
// contraction (build.py). box = {in0, in1}, Pillow's C floats, or nullptr for the default box (0, in_size) of DESIGN §13.
int resample_coefficients(uint32_t in_size, const float *box, uint32_t out_size, int resample, std::vector<int32_t> &bounds,
                          std::vector<int32_t> &coef, uint32_t &ksize);
struct ResampleFrame {
    uint64_t src;                             // byte offset of the source in the scratch: h rows of src_pitch bytes, ncomp bytes per pixel
    uint64_t inter;                           // byte offset of the horizontal pass's rows y0 .. y1 - 1 in the intermediate (tw * ncomp each)
    uint64_t h_bounds, h_coef, v_bounds, v_coef;  // byte offsets of the tables in the input buffer (16-byte aligned)
    uint64_t c_src;                           // byte offset of C in the scratch (src unless the frame reduces): c_h rows of c_pitch bytes
    // (grouped by 16 bytes so that the vertical pass reads its fields in two loads)
    uint32_t tw, th, ncomp, pass;             // the output's extent (the window's); kPassH / kPassV: the axes Pillow resamples
    uint32_t src_pitch, v_ksize, y0, plane;   // y0, y1: the rows of the source the vertical table touches (0, h: the source is trimmed
    uint32_t w, h, h_ksize, y1;               // to them); destinations: planes[4 * plane + c], in output coordinates; w x h: the source
    uint32_t stage;                           // kStageRow: a row of the source fits the shared row buffer; kStageCoef: the horizontal table fits
    uint32_t fx, fy;                          // Image.reduce's factors (1, 1: the source is C)
    uint32_t c_w, c_h, c_pitch;               // C's extent and row pitch; blocks of fx x fy pixels of C from its origin make R
};
constexpr uint32_t kStageRow = 1, kStageCoef = 2;
constexpr uint32_t kPassH = 1, kPassV = 2;
// OpenCV's filters (DESIGN §20) reuse the descriptor: a frame with kPassH | kPassV runs cv_resample_h_kernel into an intermediate
// of 4 bytes per sample and cv_resample_v_kernel, with rule 3's float tables where kPassArea is set and the two-tap int16 tables of
// rules 1 / 4 otherwise (bounds: the two rebased source indices); a frame with no pass bit sums fx x fy blocks of the source
// (rule 2; 1 x 1 for a copy) in cv_area_block_kernel.
constexpr uint32_t kPassArea = 4;
int cv_resample_coefficients(uint32_t in_size, uint32_t out_size, int table, std::vector<int32_t> &bounds, std::vector<int32_t> &coef,
                             uint32_t &ksize);
constexpr uint32_t kCvLinear = 1, kCvArea = 2, kCvBlocks = 4;  // ResampleLaunch::cv_kinds: the frame kinds of a cv batch
constexpr uint32_t kResampleRowSmem = 16 * 1024, kResampleCoefSmem = 32 * 1024;  // the shared buffers of resample_h_kernel
constexpr uint32_t kResampleRows = 8;                                            // rows of the intermediate per CTA
constexpr uint32_t kReduceRows = 4;                                              // rows of R per reduce_kernel CTA
struct ResampleLaunch {
    const ResampleFrame *frames;  // device
    uint32_t n_frames;
    uint32_t max_rows;            // largest y1 - y0 of a frame with a horizontal pass
    uint32_t max_reduce_rows;     // largest height of R of a frame that reduces (0: no reduce_kernel launch)
    uint64_t max_pixels;          // largest tw * th
    const uint8_t *input;         // the batch's input buffer (tables)
    uint8_t *scratch;
    uint8_t *inter;
    const b200jpg_plane *planes;  // device
    const b200jpg_convert *convert;  // host; null: uint8 destinations
    const float *table;           // device, with `convert`: the sample tables (FloatDst::table), the kernels' kTable instances
    uint32_t n_plain;             // frames [n_plain, n_frames) are grey frames of B200JPG_FLAG_OUTPUT_RGB: one channel in the scratch and
                                  // the intermediate, each resampled value stored to three destinations
    int resample;                 // the batch's B200JPG_RESAMPLE_*: OpenCV's filters take the cv kernels
    uint32_t cv_kinds;            // kCvLinear / kCvArea / kCvBlocks: which cv kernels some frame needs
};
int launch_resample(const ResampleLaunch &l, void *stream, int *launches);

// JPEG::DisplayRectangle into device bitmaps (bitmap_sm100.cu): the rectangle x0..x1, y0..y1 (inclusive, in the coordinates of
// the decoded samples) of every requested component goes from the decoded frame to the client's bitmap. Sample (x, y) of
// component k is src[comp[k].src_off + y * src_pitch + x * src_step] (samples of 1 or 2 bytes, `deep`) and lands at
// dst + x * bytes_per_pixel + y * bytes_per_row, as a byte or (wide_out) a native-endian 16-bit value. A component with a null
// dst, and the samples of a block whose origin (inside the rectangle) lies outside its bitmap's width x height, stay unwritten.
struct BitmapCopy {
    uint8_t *dst;
    int64_t bytes_per_pixel, bytes_per_row;
    uint32_t width, height;
    uint64_t src_off;
    uint32_t src_step, src_pitch;
};
struct BitmapRequest {
    BitmapCopy comp[4];
    int ncomp;
    int x0, x1, y0, y1;
    int deep, wide_out;
};
int launch_bitmap_copy(const BitmapRequest &r, const uint8_t *src, void *stream);
// the same from the C++ shim on the context's device: checks that every destination is device memory of that device, waits for
// the copy; returns 0 or an error code (message on the context)
int device_bitmap_copy(b200jpg_ctx *ctx, const BitmapRequest &r, const uint8_t *src);

}  // namespace b200jpg
